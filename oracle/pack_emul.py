"""A numpy restatement of the fixed-scale weight packers of the split-fp16 engines and of the epilogues that undo their
scales, held to the float64 stage oracle (``block64``'s S).  TEST INFRASTRUCTURE.

The packers are ``pack_fused`` (the expand and project weights of the stem + block-1 kernel and of the fused blocks),
``pack_tc_pointwise`` (engine 1) and the tail packer (``synergy_b200.cu``).  Each brings max |w| of a channel into
[256, 512) with a power-of-two scale 2^f, f = 9 - frexp exponent, capped at 2^117 (``channel_scale``).  The restatement
follows the kernels step by step: the activation times kActScale = 64 split into fp16 hi + lo (clamped at +-60000), the
scaled weight split the same way without the clamp, hi*hi + hi*lo + lo*hi with exact products and one fp32 rounding of
the sum (an optimistic model of the accumulator), and the fp32 epilogue factor 1 / (64 * 2^f) (for the fused expand
1 / (6 * 64 * 2^f) with the bias / 6, the hidden tensor being kept as relu6(h) / 6).

Two schemes for the fused expand: ``LAYER`` takes one scale from the largest |w| of the whole layer, ``CHANNEL`` one per
hidden channel.  The project, the tail and engine 1 scale per output channel.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import block64
from oracle.check64 import ratio

LAYER, CHANNEL = 'layer', 'channel'
SCALE_CAP = 117                       # the largest exponent of channel_scale
CAP_FLOOR = 9 - SCALE_CAP - 1         # -109: a channel max below 2^-108 packs under [256, 512)
PROJECT_K = (32, 96, 144, 192, 384, 576, 960, 320)   # the project convs of blocks 1, 2, 4, 7, 11, 14, 17 and the tail


def f32(x) -> np.ndarray:
    return np.asarray(x, np.float32)


def split(x, clamp: bool):
    """split2_f16 / split_f16_host: (hi, lo) as float64 values of fp16 numbers."""
    x = f32(x)
    if clamp:
        x = np.clip(x, np.float32(-60000), np.float32(60000))
    with np.errstate(all='ignore'):
        hi = x.astype(np.float16).astype(np.float32)
        lo = (x - hi).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def scale_exp(m) -> np.ndarray:
    """channel_exp capped at 117: f with max * 2^f in [256, 512); 0 for an all-zero channel."""
    m = np.asarray(m, np.float64)
    pos = m > 0
    return np.where(pos, np.minimum(9 - np.frexp(np.where(pos, m, 1.0))[1], SCALE_CAP), 0)


def _products(a, w, f) -> np.ndarray:
    """hi*hi + hi*lo + lo*hi of (a * 64) and (w * 2^f per column), one fp32 rounding: (M, N) fp32."""
    ah, al = split(f32(a) * np.float32(block64.ACT_SCALE), clamp=True)
    wh, wl = split(np.ldexp(f32(w), f[None, :]), clamp=False)
    return f32(ah @ wh + ah @ wl + al @ wh)


def fma(x, y, z) -> np.ndarray:
    return f32(np.asarray(x, np.float64) * np.asarray(y, np.float64) + np.asarray(z, np.float64))


def expand(a, w, b, scheme: str) -> np.ndarray:
    """The fused expand's EPI1 before its saturate, times 6: (s1 * D1 + b1 / 6) * 6 per hidden channel.  ``a`` (M, K)
    block input, ``w`` (K, N) folded fp32 weights, ``b`` (N,) folded bias."""
    w = f32(w)
    m = np.abs(w).max(axis=0)
    f = scale_exp(m) if scheme == CHANNEL else np.full(w.shape[1], scale_exp(m.max()))
    acc = _products(a, w, f)
    s1 = f32(np.float32(1.0) / (np.float32(6.0 * block64.ACT_SCALE) * f32(np.ldexp(1.0, f))))
    return fma(acc, s1[None, :], f32(b) / np.float32(6.0)).astype(np.float64) * 6.0


def per_channel(a, w, b) -> np.ndarray:
    """The per-output-channel packers' result: fmaf(D, 1 / (64 * 2^f), bias) (fused project, tail, engine 1)."""
    w = f32(w)
    f = scale_exp(np.abs(w).max(axis=0))
    acc = _products(a, w, f)
    osc = f32(np.float32(1.0) / (np.float32(block64.ACT_SCALE) * f32(np.ldexp(1.0, f))))
    return fma(acc, osc[None, :], f32(b))


def ratios(got, a, w64, b) -> np.ndarray:
    """|got - want| / S per element, want and S of ``block64``'s pointwise conv from the float64 weights ``w64``."""
    at = torch.from_numpy(np.asarray(a, np.float64))
    want, s = block64._pointwise(at, torch.zeros_like(at), torch.from_numpy(np.asarray(w64, np.float64).T),
                                 torch.from_numpy(np.asarray(b, np.float64)))
    return ratio(torch.from_numpy(np.asarray(got, np.float64)), want, s).numpy()


def relu6_rows(m: int, k: int, seed: int) -> np.ndarray:
    """(m, k) fp32 project inputs: ReLU6 outputs of Gaussian pre-activations, about half of them 0."""
    return f32(np.clip(np.random.default_rng(seed).standard_normal((m, k)) * 2.0, 0.0, 6.0))


def binade_weights(k: int, e: int, seed: int):
    """(float64 weights (k,), fp32 as the host folds them): Gaussian, max |w| = 1.5 * 2^e."""
    w = np.random.default_rng(seed).standard_normal(k)
    w = w / np.abs(w).max() * 1.5 * 2.0 ** e
    return w, f32(w)


def binade_ratio(e: int, rows: int = 1024) -> float:
    """The worst ratio of one output channel whose max |w| lies in binade 2^e, over the project Ks, with ReLU6 inputs and
    zero bias: what the per-channel packers give there."""
    worst = 0.0
    for i, k in enumerate(PROJECT_K):
        a = relu6_rows(rows, k, 100 + i)
        w64, w32 = binade_weights(k, e, 200 + i)
        got = per_channel(a, w32[:, None], np.zeros(1, np.float32))
        worst = max(worst, float(ratios(got, a, w64[:, None], np.zeros(1)).max()))
    return worst
