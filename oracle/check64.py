"""Float64 primitives the per-stage oracles share.  TEST INFRASTRUCTURE.

Every oracle (``block64``, ``gemm64``, ``mbv1_64``, ``fb64``, ``recon64``) returns ``(want, S)`` for a stage and holds it
to |got - want| <= tau * S at every element: ``ratio`` / ``worst`` measure that.  The networks' BatchNorms are folded
here in float64 from the state dict (eval mode, eps 1e-5), not from the library's folded weights.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

BN_EPS = 1e-5

Pair = Tuple[torch.Tensor, torch.Tensor]          # (value, error scale S), both float64


ABS_ALLOW = 2.0 ** -149        # one fp32 subnormal spacing: what an fp32 result cannot resolve at any scale
F32_OVERFLOW = 2.0 ** 128 - 2.0 ** 103   # round to nearest takes every |x| from here up to +-Inf


def ratio(got, want, s):
    """(|got - want| - 2^-149)+ / S per element, so that ratio <= tau means |got - want| <= tau * S + 2^-149 (0 where
    they are that close, inf where S = 0 and they differ by more).  An infinite ``got`` with the sign of ``want`` is as
    far from it as ``want`` is from the fp32 overflow threshold: Inf passes exactly where |want| >= F32_OVERFLOW - tau * S
    (and a finite ``got`` fails wherever |want| - tau * S is past it by more than FLT_MAX).  As torch tensors, or as
    numpy arrays when ``want`` is one."""
    if isinstance(want, np.ndarray):
        g = np.asarray(got, np.float64)
        with np.errstate(divide='ignore', invalid='ignore'):
            d = np.abs(g - want)
            inf_ok = np.isinf(g) & (np.sign(g) == np.sign(want))
            d = np.where(inf_ok, np.maximum(F32_OVERFLOW - np.abs(want), 0.0), np.maximum(d - ABS_ALLOW, 0.0))
            return np.where(d == 0, 0.0, d / s)
    g = got.double()
    d = (g - want).abs()
    inf_ok = torch.isinf(g) & (torch.sign(g) == torch.sign(want))
    d = torch.where(inf_ok, (F32_OVERFLOW - want.abs()).clamp_min(0.0), (d - ABS_ALLOW).clamp_min(0.0))
    return torch.where(d == 0, torch.zeros_like(d), d / s)


def worst(got, want, s) -> Tuple[float, tuple]:
    """Largest |got - want| / S and the index where it occurs."""
    r = ratio(got, want, s)
    i = int(r.argmax())
    return float(r.reshape(-1)[i]), tuple(int(v) for v in np.unravel_index(i, r.shape))


def f32_dot3(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """((a0 b0 + a1 b1) + a2 b2) over the last axis in elementwise float32, one rounding per operation and no fused
    multiply-add: the order of a kernel's unrolled three-term sum (np.linalg.norm / np.dot go through BLAS, whose order
    and FMA use depend on the host)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    with np.errstate(all='ignore'):
        return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def fold_bn(sd: Dict[str, torch.Tensor], bn_key: str, w: torch.Tensor,
            conv_bias: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The eval-mode BatchNorm ``bn_key`` folded into the conv weight ``w`` (output channels first) and its bias:
    (w * scale, (conv_bias - mean) * scale + beta), scale = gamma / sqrt(var + eps), in float64.  With no conv bias this
    rounds exactly as beta - mean * scale."""
    g = lambda k: sd[f'{bn_key}.{k}'].double()
    scale = g('weight') / torch.sqrt(g('running_var') + BN_EPS)
    cb = conv_bias.double() if conv_bias is not None else torch.zeros_like(scale)
    return w.double() * scale.view(-1, *([1] * (w.dim() - 1))), (cb - g('running_mean')) * scale + g('bias')


def strip_prefix(sd: Dict[str, torch.Tensor], prefix: str) -> Dict[str, torch.Tensor]:
    """The keys of ``sd`` that start with ``prefix``, without it; ``sd`` itself when no key does."""
    if not any(k.startswith(prefix) for k in sd):
        return sd
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def linear_heads(sd: Dict[str, torch.Tensor], keys: Sequence[str]) -> Tuple[torch.Tensor, torch.Tensor]:
    """The linear layers ``keys`` stacked along their outputs, in that order: (W, b) in float64."""
    return (torch.cat([sd[f'{k}.weight'].double() for k in keys]),
            torch.cat([sd[f'{k}.bias'].double() for k in keys]))
