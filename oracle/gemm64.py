"""Float64 per-stage oracle of the GEMM layers (ResNet-50 and the PointNet heads), with a per-element error scale.  TEST
INFRASTRUCTURE.

The contract is that of ``block64.py``: every stage is fed the exact fp32 tensor the GPU stage was fed (normally the
GPU's own output of the previous stage) and returns ``(want, S)``; a stage passes when |got - want| <= tau * S at every
element.  BatchNorm is folded here, in float64, from the state dict (``check64.fold_bn``, not the library's folded
weights).

Tensor-core stages (``tc_gemm_kernel``, csrc/kernels_gemm.cuh).  Every operand is split into fp16 hi + lo after a
power-of-two scale: row m of A by 2^e so that its max |a| (``rowmax``) lands in [2^13, 2^14), output channel n of W by
2^f so that its max |w| lands in [2^8, 2^9).  The pair holds 22 bits (2^-22 relative) while lo is a normal fp16 number;
for small operands lo falls into fp16's subnormals, whose spacing 2^-24 is absolute in scaled units.  The two bounds
meet at a scaled magnitude of 2^-24 / 2^-22 = 2^-2, i.e. at

    A:  eps_row = 2^-2 * 2^-e = 2^(E_row - 15),   E_row = floor(log2 rowmax)   (between 2^-16 and 2^-15 of the row max)
    W:  eps_n   = 2^-2 * 2^-f = 2^(E_n - 10),     E_n = floor(log2 max_k |w[n, k]|)   (between 2^-11 and 2^-10 of it)

so every product enters S as (|a| + eps_row)(|w| + eps_n): the absolute error of the subnormal lo is charged at the same
rate tau as the relative error of the pair.  The epilogue's adds enter with their absolute values:

    S = sum_k (|a_k| + eps_row)(|w_k| + eps_n) + |bias| + |addend| + |residual|

ReLU (slope <= 1) passes S on unchanged.  A row whose max is 0 is not scaled and holds exact zeros: eps_row = 0.  In conv
mode the kernel scales an output pixel's patch by the max of its in-bounds input pixels' row maxima, which is the max of
the patch itself, so eps_row is taken from the gathered patch.

CUDA-core stages (the ResNet stem, PointNet conv1 in ``small_k_layer_kernel``, the average pool) compute in fp32 and get
the fp32 form S = sum_k |a_k||w_k| + |bias|.  Copies and comparisons (max-pools, the face vector, the fp32 bit
conversion, every recorded row maximum) have no rounding and are compared bit for bit, by the tests.

Rows are what the GPU stores: one per NHWC pixel for ResNet-50, one per point (face-major, 68 per face) for the heads.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from oracle.check64 import Pair, fold_bn, linear_heads, strip_prefix, worst  # noqa: F401  (the tests' check)

PTS = 68
RESNET_PREFIX = 'I2P.backbone.'
HEADS = ('fc_ori', 'fc_shape', 'fc_exp', 'fc_tex')          # the four linear heads of ResNet-50 and MobileNetV1
FACE_VEC_LD = 2360                      # kFaceVecLd (csrc/heads_host.inl): 1024 + 1280 + 40 + 10 = 2354, padded


# ---- floors and the two forms of S ----------------------------------------------------------------------------------

def _floor_exp(m: torch.Tensor) -> torch.Tensor:
    """floor(log2 m) of magnitudes m > 0, exact for every finite fp32 value, subnormals included (frexp in float64)."""
    _, e = torch.frexp(m.double())                       # m = f * 2^e, f in [0.5, 1)
    return (e - 1).double()


def row_floor(rowmax: torch.Tensor) -> torch.Tensor:
    """eps_row per row from the true max |a| of the row."""
    rm = rowmax.double()
    return torch.where(rm > 0, torch.exp2(_floor_exp(rm) - 15), torch.zeros_like(rm))


def chan_floor(w: torch.Tensor) -> torch.Tensor:
    """eps_n per output channel of an (N, K) weight, from its fp32 values (what the library packs)."""
    m = w.float().abs().amax(dim=1).double()
    return torch.where(m > 0, torch.exp2(_floor_exp(m) - 10), torch.zeros_like(m))


def gemm(a: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], relu: bool, addend: Optional[torch.Tensor] = None,
         residual: Optional[torch.Tensor] = None, rowmax: Optional[torch.Tensor] = None) -> Pair:
    """One tensor-core stage on rows ``a`` (M, K) and weights ``w`` (N, K): (want, S), both (M, N) float64.
    ``addend`` is already broadcast to (M, N).  ``rowmax``: the row maxima the row scale comes from (default: the true
    max |a| of each row)."""
    a, w = a.double(), w.double()
    rm = a.abs().amax(dim=1) if rowmax is None else rowmax.double()
    y = a @ w.T
    s = (a.abs() + row_floor(rm)[:, None]) @ (w.abs() + chan_floor(w)[:, None]).T
    for t in (b, addend, residual):
        if t is not None:
            y, s = y + t.double(), s + t.double().abs()
    return (y.clamp_min(0.0) if relu else y), s


def simt(a: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], relu: bool) -> Pair:
    """One fp32 CUDA-core stage: (want, S = sum |a||w| + |b|)."""
    a, w = a.double(), w.double()
    y, s = a @ w.T, a.abs() @ w.abs().T
    if b is not None:
        y, s = y + b.double(), s + b.double().abs()
    return (y.clamp_min(0.0) if relu else y), s


def patches(x: torch.Tensor, ksize: int, stride: int, pad: int) -> torch.Tensor:
    """NHWC maps (B, H, W, C) -> implicit-GEMM rows (B*HO*WO, ksize*ksize*C), k = (ky * ksize + kx) * C + c."""
    x = x.double().permute(0, 3, 1, 2)
    bsz, c = x.shape[:2]
    cols = F.unfold(x, ksize, padding=pad, stride=stride)          # (B, C*k*k, L), order (c, ky, kx)
    cols = cols.view(bsz, c, ksize * ksize, -1).permute(0, 3, 2, 1)  # (B, L, tap, C)
    return cols.reshape(-1, ksize * ksize * c)


# ---- ResNet-50 (rows = NHWC pixels) ---------------------------------------------------------------------------------

def resnet_fold(sd, index: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Conv ``index`` of the 53-conv execution plan with BN folded: (W (N, K) in the GEMM's k order, bias)."""
    from synergynet_b200.backbone import resnet50_conv_keys
    sd = strip_prefix(sd, RESNET_PREFIX)
    ck, bk = resnet50_conv_keys()[index]
    w, b = fold_bn(sd, bk, sd[ck + '.weight'])
    if index == 0:                                                   # the stem keeps the OIHW order (c, ky, kx)
        return w.reshape(w.shape[0], -1), b
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1), b          # (ky, kx, c)


def resnet_stem(sd, x: torch.Tensor) -> Pair:
    """7x7/s2 conv + BN + ReLU of the NCHW image -> (B*3600, 64) rows (fp32 CUDA-core stage)."""
    w, b = resnet_fold(sd, 0)
    cols = F.unfold(x.double(), 7, padding=3, stride=2).transpose(1, 2).reshape(-1, w.shape[1])
    return simt(cols, w, b, True)


def resnet_maxpool(stem: torch.Tensor, batch: int) -> torch.Tensor:
    """MaxPool2d(3, 2, 1) of the stem rows -> (B*900, 64) fp32 rows: exact."""
    x = stem.float().view(batch, 60, 60, 64).permute(0, 3, 1, 2)
    return F.max_pool2d(x, 3, 2, 1).permute(0, 2, 3, 1).reshape(-1, 64)


def resnet_conv(sd, index: int, x: torch.Tensor, batch: int, residual: Optional[torch.Tensor] = None) -> Pair:
    """Conv ``index`` (1..52) + BN (+ the shortcut) (+ ReLU, all but the downsample) on input rows ``x`` (B*H*W, C)."""
    from synergynet_b200.backbone import resnet50_conv_keys
    w, b = resnet_fold(sd, index)
    ck = resnet50_conv_keys()[index][0]
    ksize = 3 if ck.endswith('conv2') else 1
    stride = 2 if (ck.endswith('conv2') or 'downsample' in ck) and ck.startswith(('layer2.0', 'layer3.0', 'layer4.0')) else 1
    cin = w.shape[1] // (ksize * ksize)
    hw = int(round((x.shape[0] // batch) ** 0.5))
    a = patches(x.reshape(batch, hw, hw, cin), ksize, stride, ksize // 2)
    return gemm(a, w, b, 'downsample' not in ck, residual=residual)


def avgpool(x: torch.Tensor, batch: int) -> Pair:
    """Average over the pixels of each face's rows -> (B, C) (fp32 CUDA-core stage: S = mean |x|)."""
    x = x.double().view(batch, -1, x.shape[1])
    return x.mean(dim=1), x.abs().mean(dim=1)


def resnet_heads(sd, pooled: torch.Tensor) -> Pair:
    return gemm(pooled, *linear_heads(strip_prefix(sd, RESNET_PREFIX), HEADS), False)


# ---- PointNet heads (rows = B*68 points, face-major) ---------------------------------------------------------------

def pn_fold(sd, prefix: str, conv: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """Conv1d(k=1) ``conv`` of ``prefix`` ('forwardDirection.' / 'reverseDirection.') with its BatchNorm folded."""
    sub = strip_prefix(sd, prefix)
    return fold_bn(sub, 'bn' + conv[4:], sub[conv + '.weight'][:, :, 0], sub[conv + '.bias'])


def lmk_rows(lmk: torch.Tensor) -> torch.Tensor:
    """(B, 3, 68) landmarks -> (B*68, 3) point rows."""
    return lmk.double().permute(0, 2, 1).reshape(-1, 3)


def pn_conv1(sd, prefix: str, lmk: torch.Tensor) -> Pair:
    w, b = pn_fold(sd, prefix, 'conv1')
    return simt(lmk_rows(lmk), w, b, True)


def pn_conv(sd, prefix: str, conv: str, x: torch.Tensor) -> Pair:
    """conv2..conv5, conv7..conv9 of MLP_for / conv2..conv5 of MLP_rev: GEMM + BN + ReLU on point rows."""
    w, b = pn_fold(sd, prefix, conv)
    return gemm(x, w, b, True)


def pn_pool(conv5: torch.Tensor) -> torch.Tensor:
    """Max over each face's 68 rows -> (B, C) in the input's dtype: exact."""
    return conv5.view(-1, PTS, conv5.shape[1]).amax(dim=1)


def face_vector(gmax: torch.Tensor, pool1280: torch.Tensor, params62: torch.Tensor) -> torch.Tensor:
    """conv6's per-face input [global features | avgpool | shape | expression | zero padding] as fp32: exact."""
    pad = torch.zeros((gmax.shape[0], FACE_VEC_LD - 2354), dtype=torch.float32)
    return torch.cat([gmax.float(), pool1280.float(), params62.float()[:, 12:62], pad], 1)


def conv6_face(sd, facevec: torch.Tensor) -> Pair:
    """conv6 columns [64, 2418) on the face vector, BN scale folded, no bias and no activation -> (B, 512)."""
    w, _ = pn_fold(sd, 'forwardDirection.', 'conv6')
    wf = torch.zeros((w.shape[0], FACE_VEC_LD), dtype=torch.float64)
    wf[:, :2354] = w[:, 64:]
    return gemm(facevec, wf, None, False)


def conv6_point(sd, pf: torch.Tensor, face: torch.Tensor) -> Pair:
    """conv6 columns [0, 64) on point_features + bias + the face part broadcast over the points, ReLU."""
    w, b = pn_fold(sd, 'forwardDirection.', 'conv6')
    return gemm(pf, w[:, :64], b, True, addend=face.double().repeat_interleave(PTS, dim=0))


def rev_heads(sd, glob: torch.Tensor) -> Pair:
    """conv6_1 | conv6_2 | conv6_3 (+ BN + ReLU each) of MLP_rev on the global features -> (B, 62)."""
    parts = [pn_fold(sd, 'reverseDirection.', f'conv6_{i}') for i in (1, 2, 3)]
    return gemm(glob, torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts]), True)


def residual_from_rows(conv9: torch.Tensor) -> torch.Tensor:
    """conv9's (B*68, 3) rows -> point_residual (B, 3, 68): exact."""
    return conv9.view(-1, PTS, 3).permute(0, 2, 1)


# ---- batches and faces that put the GEMM's tile edges under a check ---------------------------------------------------

TILE = 128                               # rows per CTA of tc_gemm_kernel: warpgroup 0 rows 0..63, warpgroup 1 rows 64..127
RESNET_MAPS = (900, 225, 64, 16)         # output pixels per face of the four ResNet-50 stages
RESNET_BATCHES = (13, 19, 128)
POINTNET_BATCHES = (1, 2, 37, 32)


def last_tile(m: int) -> str:
    """'full', 'wg0' (the ragged last tile keeps warpgroup 1 idle) or 'both' (both warpgroups hold rows of it)."""
    r = m % TILE
    return 'full' if r == 0 else 'wg0' if r <= 64 else 'both'


def check_resnet_batches(batches=RESNET_BATCHES) -> None:
    """At every map size the batches give a ragged last tile with only warpgroup 0 busy, one with both busy (where the
    map size allows: 64 B mod 128 is 0 or 64) and an exact multiple of 128 rows."""
    for p in RESNET_MAPS:
        kinds = {last_tile(b * p) for b in batches}
        need = {'full', 'wg0'} | ({'both'} if p % 64 else set())
        assert need <= kinds, (p, kinds)


def check_pointnet_batches(batches=POINTNET_BATCHES) -> None:
    """M = 68 B leaves: a last tile whose warpgroup 1 holds a partial first warp (68 rows: 4 in warpgroup 1), one with
    warpgroup 0 only, one with both warpgroups and more than a warp in warpgroup 1, and no ragged tile at all."""
    rems = [68 * b % TILE for b in batches]
    assert 0 in rems and any(0 < r <= 64 for r in rems), rems
    assert any(64 < r < 80 for r in rems) and any(r >= 80 for r in rems), rems


def tile_edge_faces(batch: int, maps, tile: int = TILE) -> list:
    """Faces to check at this batch of GEMMs that hold p rows per face, p each map size of ``maps``: the first and the
    last face and, at every map size, the face that straddles the edge of the last tile and the first face wholly inside
    that tile (where one fits)."""
    faces = {0, batch - 1}
    for p in maps:
        m = batch * p
        t0 = (m - 1) // tile * tile                      # first row of the last tile
        if t0 > 0:
            faces |= {(t0 - 1) // p, t0 // p}
        inside = -(-t0 // p)
        if inside < batch:
            faces.add(inside)
    return sorted(faces)


def resnet_faces(batch: int) -> list:
    """``tile_edge_faces`` over the four ResNet-50 map sizes."""
    return tile_edge_faces(batch, RESNET_MAPS)


def check_resnet_faces(batch: int, faces) -> None:
    """The faces include the last one and, per map size, one straddling a 128-row edge (when p does not divide 128 or
    128 does not divide p) and one wholly inside the ragged last tile (when a face fits in it)."""
    assert batch - 1 in faces
    for p in RESNET_MAPS:
        m = batch * p
        t0 = (m - 1) // TILE * TILE
        if p % TILE and TILE % p and m > TILE:
            assert any(f * p < e < (f + 1) * p for f in faces for e in range(TILE, m, TILE)), (batch, p)
        if m % TILE and m - t0 >= p:
            assert any(f * p >= t0 for f in faces), (batch, p)


# ---- checking --------------------------------------------------------------------------------------------------------

def rowmax_bits(x: torch.Tensor) -> torch.Tensor:
    """max |x| of every row as fp32 bit patterns (int32), what a producer must record."""
    return x.float().abs().amax(dim=1).view(torch.int32)
