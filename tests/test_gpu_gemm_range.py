"""tc_gemm_kernel across the whole fp32 range against the float64 oracle (oracle/gemm64.py), and its saturation flag.

Every case runs one syn_debug_gemm launch in plain mode and one in conv mode (3x3, stride 2, a non-square map), holds
every element to |got - want| <= TAU * S + 2^-149 (an infinite result where |want| is past the fp32 overflow threshold
by more than TAU * S), compares the recorded row maxima bit for bit, and requires the sticky saturation flag to stay 0.
The row sweep puts one 16-row group in every binade 2^-149 .. 2^127 (subnormal row maxima included), the weight sweep
one output channel in every binade over two n-ranges, and the extremes cross tiny rows with huge channels and the
reverse.  A non-finite input value must raise the flag, and every output row that does not read it keeps the bits of
the clean call.  The CPU restatement of the same scaling is tests/test_gemm_range_emulation.py.  H100 only.
"""
import numpy as np
import pytest
import torch

from oracle import gemm64, synth_model
from oracle.stage_check import TAU, check_rowmax, make_model, same_bits

pytestmark = pytest.mark.gpu

BAR = TAU['gemm64']['gemm']
K_PLAIN = 64
CONV = (3, 2, 1)                         # ksize, stride, pad
H, W, C = 9, 13, 8                       # -> 5 x 7 output maps, K = 72
HO, WO = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
WORST = {}


@pytest.fixture(scope='module')
def eng(synth_pack):
    e = make_model(synth_model.build_state_dict(0))._engine(torch.device('cuda', 0))
    e.poll_saturation(warn=False)
    yield e
    print('\n[gemm range] worst |got - want| / S: ' + '  '.join(f'{k} {v:.3e}' for k, v in WORST.items()))


def binade_block(x: int, shape, rng) -> np.ndarray:
    """Values of mixed sign whose max |v| lies in [2^x, 2^(x+1)): every row (last axis) holds its own max, an element
    2^-20 and one 2^-40 below it and two subnormals, where the binade leaves them below the max."""
    r = rng.uniform(-1.0, 1.0, shape)
    r[..., 0] = rng.uniform(1.0, 2.0, shape[:-1])
    r[..., 1] = 2.0 ** -20
    r[..., 2] = -(2.0 ** -40)
    v = r * 2.0 ** x
    v[..., 3] = 2.0 ** -140
    v[..., 4] = -(2.0 ** -149)
    return np.where(np.abs(v) < 2.0 ** (x + 1), v, 0.0)


def sweep_rows(exps, k: int, seed: int) -> torch.Tensor:
    rng = np.random.default_rng(seed)
    return torch.from_numpy(np.concatenate([binade_block(x, (16, k), rng) for x in exps])).float()


def sweep_maps(exps, seed: int) -> torch.Tensor:
    """One NHWC map (H, W, C) per binade: every input pixel's max in that binade."""
    rng = np.random.default_rng(seed)
    return torch.from_numpy(np.stack([binade_block(x, (H, W, C), rng) for x in exps])).float()


def layer(n: int, k: int, seed: int, mag: float = 1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((n, k), generator=g) / k ** 0.5 * mag, torch.zeros(n)


def rowmax_of(a: torch.Tensor, conv: bool) -> torch.Tensor:
    """What a producer records: max |a| per row (conv: per input pixel), fmaxf-style (a NaN is dropped)."""
    m = torch.nan_to_num(a.abs(), nan=0.0, posinf=float('inf'))
    return (m.amax(dim=-1).reshape(-1) if conv else m.amax(dim=1)).float()


def launch(eng, a, w, bias, conv: bool, **kw):
    """(out, rowmax_out, colmax or None) of one launch; ``a`` rows (M, K) or NHWC maps."""
    return eng.debug_gemm(w, bias, a, rowmax_of(a, conv).view(torch.int32), conv=(*CONV, HO, WO) if conv else None,
                          **kw)


def check_case(eng, name, a, w, bias, conv: bool, residual=None, addend=None, addend_group=1, act=0, colmax_group=0):
    """One launch held to the oracle; rowmax_out and (with colmax_group, after ReLU) the max-pool bit for bit."""
    out, rmo, cm = launch(eng, a, w, bias, conv, residual=residual, addend=addend, addend_group=addend_group, act=act,
                          colmax_group=colmax_group)
    assert eng.poll_saturation(warn=False) == 0, f'{name}: saturation flag on finite inputs'
    check_rowmax(out, rmo, name)
    assert not bool(torch.isnan(out).any()), f'{name}: NaN output'
    if colmax_group:
        o = out.cpu()
        full = torch.cat([o, torch.zeros((-o.shape[0] % colmax_group, o.shape[1]))]).view(-1, colmax_group, o.shape[1])
        assert same_bits(full.amax(dim=1), cm.cpu().view(torch.float32)), f'{name}: colmax'
    rows = gemm64.patches(a, *CONV) if conv else a
    add = None if addend is None else addend.repeat_interleave(addend_group, dim=0)[:rows.shape[0]]
    want, s = gemm64.gemm(rows, w, bias, act == 2, addend=add, residual=residual)
    r, ix = gemm64.worst(out.cpu(), want, s)
    key = f'{name} {"conv" if conv else "plain"}'
    WORST[key] = r
    print(f'\n[{key}] worst {r:.3e} at {ix}: got {float(out.cpu()[ix]):.6e} want {float(want[ix]):.6e}')
    assert r <= BAR, (key, r, ix)
    assert eng.poll_error() == 0
    return out


MODES = pytest.mark.parametrize('conv', [False, True], ids=['plain', 'conv'])


@MODES
def test_row_sweep_every_binade(eng, conv):
    """One 16-row group (conv: one map) per binade 2^-149 .. 2^127 against normal weights; M is not a multiple of 128,
    so the groups land in both warpgroups and in a ragged last tile.  ReLU, with the max-pool over each group (the
    PointNet max-pool, here in the epilogue that the rows outside the plain range take)."""
    exps = list(range(-149, 128))
    a = sweep_maps(exps, 1) if conv else sweep_rows(exps, K_PLAIN, 1)
    k = 9 * C if conv else K_PLAIN
    m = a.shape[0] * HO * WO if conv else a.shape[0]
    assert m % 128 > 64
    w, b = layer(40, k, 2)
    check_case(eng, 'row sweep', a, w, b, conv, act=2, colmax_group=HO * WO if conv else 16)


@MODES
def test_weight_sweep_every_binade(eng, conv):
    """Output channel maxima in every binade 2^-149 .. 2^127, a channel of subnormals only and a channel with a single
    non-zero: N = 279 spans two n-ranges.  Rows at 1, 2^-60 and 2^60."""
    k = 9 * C if conv else K_PLAIN
    g = torch.Generator().manual_seed(3)
    w = (torch.rand((279, k), generator=g, dtype=torch.float64) * 2 - 1)
    w[:, 0] = 1.5
    w[:277] *= torch.exp2(torch.arange(-149, 128, dtype=torch.float64))[:, None]
    w[:277] = torch.where(w[:277].abs() < torch.exp2(torch.arange(-148, 129, dtype=torch.float64))[:, None], w[:277], 0.0)
    w[277] = torch.randint(-2 ** 20, 2 ** 20, (k,), generator=g).double() * 2.0 ** -149
    w[278] = 0.0
    w[278, 5] = 3.0 * 2.0 ** -60
    w = w.float()
    exps = [0] * 3 + [-60] * 2 + [60] * 2
    a = sweep_maps(exps, 4) if conv else sweep_rows(exps, K_PLAIN, 4)
    check_case(eng, 'weight sweep', a, w, torch.zeros(279), conv)


def gemm_share(rows, w, sel_rows, sel_cols, bias, addend, residual):
    """min over the selected elements of (the GEMM's own part of S) / S: near 1 where nothing else is added."""
    _, s_gemm = gemm64.gemm(rows, w, None, False)
    _, s = gemm64.gemm(rows, w, bias, False, addend=addend, residual=residual)
    return float((s_gemm / s)[sel_rows][:, sel_cols].min())


@MODES
def test_opposite_extremes(eng, conv):
    """Rows at 2^-140 against channels at 2^120 and rows at 2^120 against channels at 2^-140, with bias, residual and
    addend at large and small magnitudes: results from the subnormal range to far past FLT_MAX.  Both pairings hold a
    block of elements that nothing is added to (no bias, residual or addend), so that the GEMM's own term makes up
    their S and the bar checks what the kernel computed there."""
    exps = [-140] * 3 + [120] * 3 + [-100, 100]
    a = sweep_maps(exps, 5) if conv else sweep_rows(exps, K_PLAIN, 5)
    k = 9 * C if conv else K_PLAIN
    per = HO * WO if conv else 16                                # rows per binade group
    m = a.shape[0] * per if conv else a.shape[0]
    n = 24
    g = torch.Generator().manual_seed(6)
    kinds = [2.0 ** 120, 2.0 ** -140, 1.0, 2.0 ** 60, 2.0 ** -60, 2.0 ** 127]
    w = (torch.rand((n, k), generator=g) * 2 - 1) * torch.tensor(kinds * 4)[:, None]
    bias = torch.tensor([0.0, 0.0, 0.0, 3.0, 2.0 ** -149, -1.0] + [2.0 ** -130, -(2.0 ** 100), 0.0, 3.0, 2.0 ** -149, -1.0] * 3)
    res = torch.randn((m, n), generator=g) * torch.exp2(torch.randint(-140, 120, (m, 1), generator=g).float())
    res[::2] = 0.0                                               # even rows: no residual
    add = torch.randn((-(-m // 8), n), generator=g) * torch.exp2(torch.randint(-140, 120, (1, n), generator=g).float())
    add[:, :6] = 0.0                                             # channels 0..5: no addend
    rows = gemm64.patches(a, *CONV) if conv else a
    add_rows = add.repeat_interleave(8, dim=0)[:m]
    even = lambda lo, hi: torch.arange(lo + lo % 2, hi, 2)     # the rows with no residual
    tiny, huge = even(0, 3 * per), even(3 * per, 6 * per)
    for r_sel, col in ((tiny, 0), (huge, 1)):                    # 2^-140 rows x 2^120 channel, 2^120 rows x 2^-140
        assert len(r_sel) > 0
        assert gemm_share(rows, w, r_sel, [col], bias, add_rows, res) > 0.99, (conv, col)
    out = check_case(eng, 'extremes', a, w, bias, conv, residual=res, addend=add, addend_group=8)
    o = out.cpu()
    assert bool(torch.isinf(o).any()), 'no output past FLT_MAX'
    assert bool(((o != 0) & (o.abs() < 2.0 ** -126)).any()), 'no output in the subnormal range'
    want, s = gemm64.gemm(rows, w, None, False)
    for r_sel, col, tag in ((tiny, 0, 'rows 2^-140 x channel 2^120'), (huge, 1, 'rows 2^120 x channel 2^-140')):
        got = o[r_sel][:, [col]]
        assert bool((got != 0).all() & torch.isfinite(got).all()), tag    # normal results, not a bias or a clamp
        r, ix = gemm64.worst(got, want[r_sel][:, [col]], s[r_sel][:, [col]])
        WORST[f'{tag} {"conv" if conv else "plain"}'] = r
        assert r <= BAR, (tag, r, ix)


@MODES
@pytest.mark.parametrize('bad', [float('nan'), float('inf'), -float('inf')], ids=['nan', 'inf', '-inf'])
def test_nonfinite_input_raises_the_flag(eng, conv, bad):
    """One non-finite element of one row (conv: one input pixel, which four output rows read): the flag is raised by
    that call alone, and every output row whose inputs are all finite keeps the clean call's bits."""
    k = 9 * C if conv else K_PLAIN
    a = sweep_maps([0, 3, -2], 7) if conv else sweep_rows([0, 3, -2, 5, 40, -40, 1, 0, 2, 0, 1, 7, 0], K_PLAIN, 7)
    w, b = layer(48, k, 8)
    clean = launch(eng, a, w, b, conv)[0]
    assert eng.poll_saturation(warn=False) == 0
    poisoned = a.clone()
    if conv:
        poisoned[1, 5, 7, 3] = bad
        mask = torch.zeros(a.shape[:3] + (1,))
        mask[1, 5, 7, 0] = 1.0
        touched = gemm64.patches(mask, *CONV).abs().amax(dim=1) > 0
        assert int(touched.sum()) == 4                           # stride 2: an odd pixel is read by 2 x 2 output pixels
    else:
        poisoned[100, 37] = bad
        touched = torch.zeros(a.shape[0], dtype=torch.bool)
        touched[100] = True
    out = launch(eng, poisoned, w, b, conv)[0]
    assert eng.poll_saturation(warn=False) == 1
    assert eng.poll_saturation(warn=False) == 0                 # cleared by the poll
    keep = ~touched
    assert same_bits(out.cpu()[keep], clean.cpu()[keep])
    assert eng.poll_error() == 0
