"""A numpy restatement of tc_gemm_kernel's scaling (csrc/kernels_gemm.cuh) held to the float64 oracle (oracle/gemm64.py)
across the whole fp32 range, without a GPU.

The emulation follows the kernel step by step: the row exponent read from the row maximum's fp32 bits, the channel
scale the host packs the weights with, the clamped fp16 hi/lo split, hi*hi + hi*lo + lo*hi (exact products, one fp32
rounding of the sum), and the epilogue's multiply order.  ``OLD`` is the scheme before the range fix: the row exponent
clamped to [-100, 100] (subnormal rows unscaled) and the channel scale a float that overflows below 2^-119.  ``NEW`` is
the kernel's.  The old scheme must fail the oracle where the range fix says it does, the new one must pass everywhere,
and in range the two must agree bit for bit.
"""
import numpy as np
import pytest
import torch

from oracle import gemm64
from oracle.check64 import ratio
from oracle.stage_check import TAU

BAR = TAU['gemm64']['gemm']
OLD, NEW = 'old', 'new'
PLAIN = 100                                   # kGmPlainExp


def f32(x):
    return np.asarray(x, np.float32)


def pow2(e) -> np.ndarray:
    """2^e as fp32 for integer e in [-149, 127] (subnormal below -126)."""
    return f32(np.ldexp(1.0, np.asarray(e, np.int64)))


def fma(x, y, z) -> np.ndarray:
    """fmaf: the product of two fp32 values is exact in float64; the sum is rounded once more (to fp32)."""
    with np.errstate(all='ignore'):
        return f32(np.asarray(x, np.float64) * np.asarray(y, np.float64) + np.asarray(z, np.float64))


def floor_log2(m: np.ndarray) -> np.ndarray:
    return np.frexp(np.asarray(m, np.float64))[1].astype(np.int64) - 1


def row_exp(rowmax: np.ndarray, scheme: str) -> np.ndarray:
    """gemm_row_exp: e with rowmax * 2^e in [2^13, 2^14); 0 for a zero or non-finite row."""
    rowmax = f32(rowmax)
    fin = np.isfinite(rowmax) & (rowmax > 0)
    e = np.where(fin, 13 - floor_log2(np.where(fin, rowmax, 1.0)), 0)
    if scheme == OLD:
        normal = rowmax >= np.float32(2.0 ** -126)
        e = np.where(normal & fin, np.clip(e, -PLAIN, PLAIN), 0)
    return e


def split(x: np.ndarray, clamp: bool = True):
    """split2_f16 / split_f16_host: (hi, lo) as fp32 values of fp16 numbers.  The clamp is fminf(fmaxf(x, -60000),
    60000): NaN becomes -60000."""
    x = f32(x)
    if clamp:
        x = np.where(np.isnan(x), np.float32(-60000), np.clip(x, np.float32(-60000), np.float32(60000)))
    with np.errstate(all='ignore'):
        hi = x.astype(np.float16).astype(np.float32)
        lo = (x - hi).astype(np.float16).astype(np.float32)
    return hi, lo


def pack(w: np.ndarray, scheme: str):
    """build_gemm_layer: the scaled weights (N, K) fp32 and the channel exponent g (NEW) or fp32 oscale (OLD)."""
    m = np.abs(w).max(axis=1)
    f = np.where(m > 0, 9 - (floor_log2(np.where(m > 0, m, 1.0)) + 1), 0)
    if scheme == OLD:
        with np.errstate(all='ignore'):
            ws = f32(np.ldexp(1.0, f))                               # ldexpf(1, 9 - ex): +Inf past 2^127
            return w * ws[:, None], np.float32(1.0) / ws
    return f32(np.ldexp(w.astype(np.float64), f[:, None])), -f


def emulate(a: np.ndarray, w: np.ndarray, bias: np.ndarray, scheme: str) -> np.ndarray:
    """out (M, N) fp32 of one plain-mode launch, no activation."""
    a, w, bias = f32(a), f32(w), f32(bias)
    e = row_exp(np.abs(a).max(axis=1), scheme)
    with np.errstate(all='ignore'):
        if scheme == OLD:
            xs = a * pow2(e)[:, None]
        else:                                                         # 2^e as two exact factors where e > 126
            xs = (a * pow2(np.maximum(e - 126, 0))[:, None]) * pow2(np.minimum(e, 126))[:, None]
        ah, al = split(xs)
        wp, chan = pack(w, scheme)
        wh, wl = split(wp, clamp=False)
        acc = f32(ah.astype(np.float64) @ wh.T.astype(np.float64) + ah.astype(np.float64) @ wl.T.astype(np.float64)
                  + al.astype(np.float64) @ wh.T.astype(np.float64))
    if scheme == OLD:
        with np.errstate(all='ignore'):
            x = acc * pow2(-e)[:, None]
        return fma(x, chan[None, :], bias[None, :])
    g = chan
    plain_rows = (np.abs(e) <= PLAIN) & bool((g >= -149).all())
    with np.errstate(all='ignore'):
        x = acc * pow2(np.where(plain_rows, -e, 0))[:, None]
    plain = fma(x, pow2(np.maximum(g, -149))[None, :], bias[None, :])
    c = g[None, :] - e[:, None]                                       # gemm_wide_out
    c2 = np.clip(c, -149, 127)
    c1 = np.clip(c - c2, -126, 127)
    with np.errstate(all='ignore'):
        wide = fma(acc * pow2(c1), pow2(c2), bias[None, :])
    return np.where(plain_rows[:, None], plain, wide)


def ratios(a, w, bias, scheme) -> np.ndarray:
    got = emulate(a, w, bias, scheme)
    want, s = gemm64.gemm(torch.from_numpy(f32(a)), torch.from_numpy(f32(w)), torch.from_numpy(f32(bias)), False)
    return ratio(torch.from_numpy(got), want, s).numpy()


def passes(r: np.ndarray) -> bool:
    return bool((r <= BAR).all())                                     # NaN fails


def binade_rows(exps, k: int, seed: int) -> np.ndarray:
    """Rows whose max lies in [2^x, 2^(x+1)) for each x of ``exps`` (16 rows each), mixed sign, each row also holding
    elements 2^-20 and 2^-40 below its max and, where the binade allows, subnormals."""
    rng = np.random.default_rng(seed)
    rows = []
    for x in exps:
        r = rng.uniform(-1.0, 1.0, (16, k))
        r[:, 0] = rng.uniform(1.0, 2.0, 16)
        r[:, 1] = 2.0 ** -20
        r[:, 2] = -(2.0 ** -40)
        v = r * 2.0 ** x
        v[:, 3] = 2.0 ** -140
        v[:, 4] = -(2.0 ** -149)
        rows.append(np.where(np.abs(v) <= 2.0 ** (x + 1), v, 0.0))
    return f32(np.concatenate(rows))


def normal_layer(n: int, k: int, seed: int, mag: float = 1.0):
    rng = np.random.default_rng(seed)
    return f32(rng.standard_normal((n, k)) / k ** 0.5 * mag), np.zeros(n, np.float32)


def tiny_channel_layer(n: int, k: int, seed: int, binade: int):
    """Normal weights, one channel whose max lies in [2^binade, 2^(binade+1)), one with only subnormals."""
    w, b = normal_layer(n, k, seed)
    rng = np.random.default_rng(seed + 1)
    w[3] = f32(rng.uniform(-1.0, 1.0, k) * 2.0 ** binade)
    w[3, 0] = f32(1.5 * 2.0 ** binade)
    w[5] = f32(rng.integers(-2 ** 20, 2 ** 20, k) * 2.0 ** -149)
    return w, b


# (name, rows, weights, bias): the cases the range fix names, where the old scheme must fail
FAILS_TODAY = {
    'row 2^-118': lambda: (binade_rows([-118], 64, 1), *normal_layer(8, 64, 2)),
    'row 2^116': lambda: (binade_rows([116], 64, 3), *normal_layer(8, 64, 4)),
    'subnormal row': lambda: (binade_rows([-140], 64, 5), *normal_layer(8, 64, 6, mag=2.0 ** 100)),
    'channel 2^-125': lambda: (binade_rows([0], 64, 7), *tiny_channel_layer(8, 64, 8, -125)),
}


@pytest.mark.parametrize('scheme', [OLD, NEW])
@pytest.mark.parametrize('case', sorted(FAILS_TODAY))
def test_range_edges_fail_today_and_pass_fixed(case, scheme):
    r = ratios(*FAILS_TODAY[case](), scheme)
    worst = float(np.nan_to_num(r, nan=np.inf).max())
    print(f'\n[{scheme} {case}] worst {worst:.3e}')
    if scheme == OLD:
        assert not passes(r), (case, worst)
    else:
        assert passes(r), (case, worst)


def test_row_sweep_every_binade():
    """One 16-row group per binade 2^-149 .. 2^127 against normal weights, and the same rows against weights at
    2^+100 and 2^-100: the fixed scheme holds every element to the bar."""
    a = binade_rows(range(-149, 128), 64, 11)
    for mag in (1.0, 2.0 ** 100, 2.0 ** -100):
        w, b = normal_layer(16, 64, 12, mag)
        r = ratios(a, w, b, NEW)
        assert passes(r), (mag, float(r.max()), np.unravel_index(r.argmax(), r.shape))


def test_weight_sweep_every_binade():
    """Channel maxima in every binade 2^-149 .. 2^127, a subnormal-only channel and a single non-zero, against rows at
    1, 2^-100 and 2^+100."""
    k = 64
    rng = np.random.default_rng(21)
    w = rng.uniform(-1.0, 1.0, (279, k))
    w[:, 0] = 1.5
    w *= np.ldexp(1.0, np.arange(-149, 130))[:, None]
    w[:277] = np.where(np.abs(w[:277]) < 2.0 ** (np.arange(-149, 128)[:, None] + 1), w[:277], 0.0)
    w[277] = rng.integers(-2 ** 20, 2 ** 20, k) * 2.0 ** -149
    w[278] = 0.0
    w[278, 17] = 3.0 * 2.0 ** -60
    w = f32(w)
    b = np.zeros(w.shape[0], np.float32)
    for x in (0, -100, 100):
        a = binade_rows([x], k, 22)
        r = ratios(a, w, b, NEW)
        assert passes(r), (x, float(r.max()), np.unravel_index(r.argmax(), r.shape))


def test_opposite_extremes_and_overflow():
    """Rows at 2^-140 against channels at 2^120 and the reverse: results from the subnormal range to past FLT_MAX
    (which must become Inf), every element under the bar.  The two extreme channels carry no bias, so the GEMM's own
    term is their whole S and the bar checks what the scheme computed there."""
    k = 64
    rng = np.random.default_rng(31)
    rows = np.concatenate([binade_rows([-140], k, 32), binade_rows([120], k, 33), binade_rows([100], k, 34)])
    w = f32(rng.uniform(-1.0, 1.0, (4, k)) * np.array([2.0 ** 120, 2.0 ** -140, 2.0 ** -20, 2.0 ** 30])[:, None])
    bias = f32([0.0, 0.0, 2.0 ** -130, 3.0])
    got = emulate(rows, w, bias, NEW)
    assert np.all(np.isfinite(got[:16, 0]) & (got[:16, 0] != 0)) and np.all(np.isfinite(got[16:32, 1]) & (got[16:32, 1] != 0))
    assert np.isinf(got[16:32, 3]).any(), 'a case past FLT_MAX'
    assert (np.abs(got[:, 1]) < 2.0 ** -126).any() or (np.abs(got[:16, 2]) < 2.0 ** -126).any(), 'a subnormal case'
    r = ratios(rows, w, bias, NEW)
    assert passes(r), (float(r.max()), np.unravel_index(r.argmax(), r.shape))


def test_in_range_bits_do_not_change():
    """Rows with |e| <= 100 against channels with a finite scale: the fixed scheme computes the old bits."""
    a = binade_rows(range(-87, 114, 7), 64, 41)
    w = np.delete(tiny_channel_layer(24, 64, 42, -100)[0], 5, axis=0)     # channel 3 at 2^-100; no subnormal channel
    b = f32(np.random.default_rng(43).standard_normal(23))
    assert np.array_equal(emulate(a, w, b, OLD).view(np.int32), emulate(a, w, b, NEW).view(np.int32))


def test_emulation_matches_the_oracle_bar_in_range():
    """The restatement itself: random rows and weights in range pass under both schemes."""
    rng = np.random.default_rng(51)
    a = f32(rng.standard_normal((64, 96)) * np.ldexp(1.0, rng.integers(-6, 5, 96)))
    w, _ = normal_layer(40, 96, 52)
    b = f32(rng.standard_normal(40))
    for scheme in (OLD, NEW):
        assert passes(ratios(a, w, b, scheme)), scheme
