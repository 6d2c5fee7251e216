"""Float64 per-stage oracle of the MobileNetV1 backbones, with a per-element error scale.  TEST INFRASTRUCTURE.

The contract is that of ``gemm64.py`` (whose docstring defines both forms of S): every stage is fed the exact fp32 tensor
the GPU stage was fed (normally the GPU's own output of the previous stage) and returns ``(want, S)``; a stage passes when
|got - want| <= tau * S at every element.  BatchNorm is folded here, in float64, from the state dict
(``check64.fold_bn``).

  * conv_sep (1x1) and the heads run on ``tc_gemm_kernel``: the split-GEMM form of ``gemm64.gemm``, with the row scale
    taken from the true max |a| of each row -- which is what the depthwise kernel and the pool record.
  * the stem (K = 27) and the depthwise convs (K = 9) run in fp32 on CUDA cores: S = sum_k |a_k||w_k| + |b|.
  * the average pool: ``gemm64.avgpool``.

Rows are what the GPU stores: one per NHWC pixel, or one per face after the pool.  Stage numbering is that of
``syn_debug_mbv1_until``: 0 stem, 2j - 1 / 2j conv_dw / conv_sep of block j = 1..13, 27 pool, 28 heads.
"""
from __future__ import annotations

import math
from typing import List, Tuple

import torch
import torch.nn.functional as F

from oracle import gemm64
from oracle.check64 import Pair, fold_bn, linear_heads, strip_prefix
from oracle.gemm64 import HEADS

PREFIX = 'I2P.backbone.'
NUM_STAGES = 29


def widen_of(arch: str) -> float:
    from synergynet_b200.backbone import MBV1_WIDTHS
    return MBV1_WIDTHS[arch]


def stage_table(arch: str) -> List[tuple]:
    """(cin, cout, ksize, stride, groups, h_in, h_out) of the 27 convolutions, from the reference's layer list
    (mobilenetv1_backbone.py:57-82) and PyTorch's conv arithmetic (padding 1 for every 3x3)."""
    from synergynet_b200.backbone import MBV1_BLOCKS
    w = widen_of(arch)
    c0 = int(32 * w)
    out = [(3, c0, 3, 2, 1, 120, (120 + 2 - 3) // 2 + 1)]
    cin, h = c0, out[0][6]
    for _, cout, stride in MBV1_BLOCKS:
        ho = (h + 2 - 3) // stride + 1
        out.append((cin, cin, 3, stride, cin, h, ho))
        out.append((cin, int(cout * w), 1, 1, 1, ho, ho))
        cin, h = int(cout * w), ho
    return out


def fold(sd, index: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Conv ``index`` of the 27-conv plan with BN folded in float64: (W (cout, cin/groups, k, k), bias)."""
    from synergynet_b200.backbone import mobilenet_v1_conv_keys
    sd = strip_prefix(sd, PREFIX)
    ck, bk = mobilenet_v1_conv_keys()[index]
    return fold_bn(sd, bk, sd[ck + '.weight'])


def _nchw(rows: torch.Tensor, batch: int) -> torch.Tensor:
    hw = int(round(math.sqrt(rows.shape[0] // batch)))
    return rows.double().view(batch, hw, hw, rows.shape[1]).permute(0, 3, 1, 2)


def _rows(x: torch.Tensor) -> torch.Tensor:
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])


def stem(sd, x: torch.Tensor) -> Pair:
    """conv1 3x3/s2/p1 + bn1 + ReLU of the NCHW crops -> (B*3600, C0) rows (fp32 CUDA-core stage)."""
    w, b = fold(sd, 0)
    cols = F.unfold(x.double(), 3, padding=1, stride=2).transpose(1, 2).reshape(-1, 27)
    return gemm64.simt(cols, w.reshape(w.shape[0], -1), b, True)


def depthwise(sd, index: int, x: torch.Tensor, batch: int) -> Pair:
    """conv_dw (index odd) + bn_dw + ReLU on input rows ``x`` (B*H*W, C) -> (B*HO*WO, C) (fp32 CUDA-core stage)."""
    from synergynet_b200.backbone import MBV1_BLOCKS
    w, b = fold(sd, index)
    stride = MBV1_BLOCKS[(index - 1) // 2][2]                          # dw2_2, dw3_2, dw4_2, dw5_6: stride 2
    a = _nchw(x, batch)
    c = a.shape[1]
    y = F.conv2d(a, w, None, stride, 1, 1, c) + b.view(1, -1, 1, 1)
    s = F.conv2d(a.abs(), w.abs(), None, stride, 1, 1, c) + b.abs().view(1, -1, 1, 1)
    return _rows(y).clamp_min(0.0), _rows(s)


def pointwise(sd, index: int, x: torch.Tensor) -> Pair:
    """conv_sep (index even, >= 2) + bn_sep + ReLU on the depthwise output rows (tensor-core stage)."""
    w, b = fold(sd, index)
    return gemm64.gemm(x, w.reshape(w.shape[0], -1), b, True)


def heads(sd, pooled: torch.Tensor) -> Pair:
    """fc_ori | fc_shape | fc_exp | fc_tex on the pooled features -> (B, 102) (tensor-core stage, no activation)."""
    return gemm64.gemm(pooled, *linear_heads(strip_prefix(sd, PREFIX), HEADS), False)


def stage(sd, index: int, inp: torch.Tensor, batch: int) -> Pair:
    """Stage ``index`` of syn_debug_mbv1_until on its input: the NCHW crops for 0, the previous stage's rows otherwise."""
    if index == 0:
        return stem(sd, inp)
    if index <= 26:
        return depthwise(sd, index, inp, batch) if index % 2 == 1 else pointwise(sd, index, inp)
    return gemm64.avgpool(inp, batch) if index == 27 else heads(sd, inp)


@torch.no_grad()
def forward64(sd, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The whole network in float64 on crops ``x`` (B,3,120,120): (out102, pooled), what MobileNet.forward computes."""
    b = x.shape[0]
    cur = stem(sd, x)[0]
    for i in range(1, 27):
        cur = stage(sd, i, cur, b)[0]
    pooled = gemm64.avgpool(cur, b)[0]
    return heads(sd, pooled)[0], pooled


# ---- batches and faces that put the tile edges under a check ----------------------------------------------------------

MAPS = (3600, 900, 225, 64, 16)          # output pixels per face of the five map sizes (60, 30, 15, 8, 4)
BATCHES = (2, 33, 128)


def dw_rows(ho: int) -> int:
    """Output rows per CTA of dw3x3_kernel (csrc/mbv1_host.inl dw_tile): about 128 pixels."""
    return min(ho, -(-128 // ho))


def last_tile_kinds(p: int, batches) -> set:
    """Shapes of the GEMM's last 128-row tile over the batches at map size p: 'min' (the fewest rows a ragged tile can
    hold there, gcd(p, 128): 1 row at 225 pixels), 'full' (128 rows: no ragged tile) and 'mid' (anything in between)."""
    g = math.gcd(p, gemm64.TILE)
    kinds = set()
    for b in batches:
        r = b * p % gemm64.TILE
        kinds.add('full' if r == 0 else 'min' if r == g else 'mid')
    return kinds


def check_mbv1_batches(batches=BATCHES) -> None:
    """At every map size the batches put the GEMM's last 128-row tile at its fewest rows, at 128 rows and in between
    (where the map size allows a value in between), and they run the depthwise kernel's last partial band (a band of
    fewer than dw_rows(HO) output rows, at HO = 15) on the last face of each batch, which the checked faces include."""
    for p in MAPS:
        g = math.gcd(p, gemm64.TILE)
        need = {'min', 'full'} | ({'mid'} if gemm64.TILE // g > 2 else set())
        kinds = last_tile_kinds(p, batches)
        assert need <= kinds, (p, kinds)
    partial = [ho for ho in (60, 30, 15, 8, 4) if ho % dw_rows(ho)]
    assert partial, 'no map size has a partial depthwise band'
    assert batches and all(b - 1 in faces(b) for b in batches), 'no batch runs a last partial band under the check'


def faces(batch: int) -> list:
    """``gemm64.tile_edge_faces`` over the five MobileNetV1 map sizes."""
    return gemm64.tile_edge_faces(batch, MAPS)
