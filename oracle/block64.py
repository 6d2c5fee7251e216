"""Float64 per-stage oracle of the MobileNetV2 backbone, with a per-element error scale.  TEST INFRASTRUCTURE.

``reference_port.mobilenetv2_forward`` is the fp32 restatement pinned to the reference's golden vectors and is chained
from the image.  This module answers a different question: given the exact fp32 tensor a GPU stage was fed, what
should that one stage have returned, and how much rounding may it carry?  Each stage here takes its input as given
(normally the GPU's own output of the previous stage), so errors do not accumulate and the check can be tight and per
element:

    |got - want| <= tau * S

``S`` is the first-order running error bound of the stage.  At every rounded step it adds the absolute values of all
terms that enter that step (|w| * |a| summed, |bias|, the skip); the S of an earlier step inside the same stage is
carried through |W| and the depthwise |taps| together with the magnitudes, and ReLU6 (slope <= 1) passes S on
unchanged.  The magnitudes fed to the next step are those of the actual clamped activations.

Fixed-scale floor.  The split-fp16 tensor-core engines store every activation operand as ``x * kActScale`` split into
fp16 hi + lo (``tc_common.cuh``, kActScale = 64).  The pair holds 22 bits (2^-22 relative) while lo is a normal fp16
number; for small x, lo falls into fp16's subnormals, whose spacing 2^-24 is absolute, i.e. 2^-24 / kActScale in
activation units.  The two bounds meet at |x| = ACT_FLOOR = 2^-24 / kActScale / 2^-22 = 2^-8, so every operand enters
S as |x| + ACT_FLOOR: the fixed-scale absolute error is charged at the same rate tau as the relative one.

BatchNorm is folded here, in float64, from the state dict (``check64.fold_bn``, not the library's folded weights).
Pointwise convs are matmuls over NHWC and the depthwise 3x3 is nine shifted multiply-adds on a zero-padded tensor.
Tensors are NHWC, the layout ``syn_debug_forward_until`` returns; the stem takes the NCHW image.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from oracle.check64 import Pair, fold_bn, linear_heads, worst  # noqa: F401  (worst: the check the stage tests apply)
from synergynet_b200.backbone import conv_plan

ACT_SCALE = 64.0                         # tc::kActScale (csrc/tc_common.cuh)
ACT_FLOOR = 2.0 ** -24 / ACT_SCALE / 2.0 ** -22
PREFIX = 'I2P.backbone.'

_PLAN = conv_plan()


def fold(sd: Dict[str, torch.Tensor], index: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Conv ``index`` of the plan with its eval-mode BatchNorm folded in float64 -> (weight, bias)."""
    spec = _PLAN[index]
    return fold_bn(sd, PREFIX + spec.bn_key, sd[PREFIX + spec.conv_key + '.weight'])


def _pointwise(a: torch.Tensor, s_a: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> Pair:
    w2 = w.reshape(w.shape[0], -1)
    y = a @ w2.T + b
    s = (a.abs() + s_a + ACT_FLOOR) @ w2.abs().T + b.abs()
    return y, s


def _depthwise(a: torch.Tensor, s_a: torch.Tensor, w: torch.Tensor, b: torch.Tensor, stride: int) -> Pair:
    n, h, wd, c = a.shape
    ho, wo = (h - 1) // stride + 1, (wd - 1) // stride + 1
    ap = F.pad(a, (0, 0, 1, 1, 1, 1))
    mp = F.pad(a.abs() + s_a + ACT_FLOOR, (0, 0, 1, 1, 1, 1))
    y = torch.zeros((n, ho, wo, c), dtype=torch.float64)
    s = torch.zeros_like(y)
    for dy in range(3):
        for dx in range(3):
            t = w[:, 0, dy, dx]
            win = (slice(None), slice(dy, dy + stride * (ho - 1) + 1, stride),
                   slice(dx, dx + stride * (wo - 1) + 1, stride), slice(None))
            y += ap[win] * t
            s += mp[win] * t.abs()
    return y + b, s + b.abs()


def _stem(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> Pair:
    """3x3 stride-2 conv of the NCHW image as one matmul over (c, dy, dx) patches."""
    xp = F.pad(x, (1, 1, 1, 1))
    ho = (x.shape[2] - 1) // 2 + 1
    cols = [xp[:, :, dy:dy + 2 * (ho - 1) + 1:2, dx:dx + 2 * (ho - 1) + 1:2] for dy in range(3) for dx in range(3)]
    patches = torch.stack(cols, -1).permute(0, 2, 3, 1, 4).reshape(x.shape[0], ho, ho, -1)
    return _pointwise(patches, torch.zeros_like(patches), w, b)


def _conv(sd, index: int, x: torch.Tensor, s_x: torch.Tensor, skip: Optional[torch.Tensor]) -> Pair:
    spec = _PLAN[index]
    w, b = fold(sd, index)
    if spec.kind == 'stem':
        y, s = _stem(x, w, b)
    elif spec.kind == 'dw':
        y, s = _depthwise(x, s_x, w, b, spec.stride)
    else:
        y, s = _pointwise(x, s_x, w, b)
    if spec.relu6:
        y = y.clamp(0.0, 6.0)
    if skip is not None:
        y, s = y + skip, s + skip.abs()
    return y, s


def conv(sd: Dict[str, torch.Tensor], index: int, x: torch.Tensor, skip: Optional[torch.Tensor] = None) -> Pair:
    """One conv + BN (+ ReLU6) (+ the skip, for a residual project conv) from its exact input: the stages of the
    unfused engines.  ``x`` is NHWC (the NCHW image for index 0); returns NHWC (value, S)."""
    x = x.double()
    return _conv(sd, index, x, torch.zeros_like(x), None if skip is None else skip.double())


def block(sd: Dict[str, torch.Tensor], b: int, x: torch.Tensor, skip: Optional[torch.Tensor] = None) -> Pair:
    """Inverted-residual block ``b`` (1..17) as one stage, the unit of the fused engine; block 1 includes the stem and
    takes the NCHW image.  The rounding of the hidden tensors inside the block is carried in S.  ``skip`` is what a
    residual block adds to its output (default ``x``): the fused kernel adds its fp32 input even where the expand GEMM
    read a clamped copy of it."""
    x = x.double()
    skip = x if skip is None else skip.double()
    idx = [s.index for s in _PLAN if s.block == b or (b == 1 and s.kind == 'stem')]
    y, s = x, torch.zeros_like(x)
    for i in idx:
        y, s = _conv(sd, i, y, s, skip if _PLAN[i].residual else None)
    return y, s


def avgpool(x: torch.Tensor, s_x: Optional[torch.Tensor] = None) -> Pair:
    """Average over the pixels of an NHWC tensor -> (N, C)."""
    x = x.double()
    s = x.abs() + ACT_FLOOR if s_x is None else x.abs() + s_x + ACT_FLOOR
    return x.mean(dim=(1, 2)), s.mean(dim=(1, 2))


def tail(sd: Dict[str, torch.Tensor], x: torch.Tensor) -> Pair:
    """Last conv + ReLU6 + average pool (the fused engine's tail kernel) from the block-17 output."""
    return avgpool(*conv(sd, len(_PLAN) - 1, x))


def heads(sd: Dict[str, torch.Tensor], pool: torch.Tensor) -> Pair:
    """The three linear heads on the pooled feature -> (N, 62) params."""
    pool = pool.double()
    w, b = linear_heads(sd, [f'{PREFIX}{k}.1' for k in ('classifier_ori', 'classifier_shape', 'classifier_exp')])
    return _pointwise(pool, torch.zeros_like(pool), w, b)
