"""Float64 per-stage oracle of the seven ResNet backbones, with a per-element error scale.  TEST INFRASTRUCTURE.

``gemm64`` holds ResNet-50's stages; this module is the same oracle for any arch of ``backbone.RESNET_ARCHS``
(resnet18 / 34 with BasicBlock, resnet50 / 101 / 152 and wide_resnet50_2 / wide_resnet101_2 with Bottleneck).  Every
function takes ``arch`` and defaults to resnet50, where it computes what the ``gemm64.resnet_*`` functions compute.  The
contract is that of ``gemm64`` (whose docstring defines both forms of S): every stage is fed the exact fp32 tensor the GPU
stage was fed and returns ``(want, S)``; a stage passes when |got - want| <= tau * S at every element.

  * every convolution after the stem and the heads run on ``tc_gemm_kernel``: the split-GEMM form of ``gemm64.gemm``;
  * the stem (K = 147) and the average pool are fp32 CUDA-core stages: ``gemm64.simt`` and ``gemm64.avgpool``;
  * the max-pool is exact.

Stage numbering is that of ``syn_debug_resnet_until``: 0 stem, 1 max-pool, 1 + i conv i (state-dict order, a block's
downsample before the conv that adds it), n + 1 avgpool, n + 2 heads, n = the number of convs.
"""
from __future__ import annotations

import functools
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F

from oracle import gemm64
from oracle.check64 import BN_EPS, Pair, fold_bn, linear_heads, strip_prefix
from oracle.gemm64 import HEADS, RESNET_PREFIX


@functools.lru_cache(maxsize=None)
def conv_keys(arch: str = 'resnet50') -> Tuple[Tuple[str, str], ...]:
    from synergynet_b200.backbone import resnet_conv_keys
    return tuple(resnet_conv_keys(arch))


@functools.lru_cache(maxsize=None)
def stage_table(arch: str = 'resnet50') -> Tuple[tuple, ...]:
    """(cin, cout, ksize, stride, h_in, h_out, residual) of every convolution, from the reference's layer list
    (resnet_backbone.py:50-225) and PyTorch's conv arithmetic: the 3x3 convs and the stem are padded (1, 3), the 1x1 are
    not.  ``residual``: the conv adds the block's shortcut (BasicBlock conv2, Bottleneck conv3)."""
    from synergynet_b200 import backbone
    m = getattr(backbone, arch)()
    keys = conv_keys(arch)
    geo = lambda i: (lambda c: (c.in_channels, c.out_channels, c.kernel_size[0], c.stride[0]))(m.get_submodule(keys[i][0]))
    out = [(3, 64, 7, 2, 120, (120 + 6 - 7) // 2 + 1, False)] + [None] * (len(keys) - 1)
    h = (out[0][5] + 2 - 3) // 2 + 1                                    # the max-pool: 60 -> 30
    for inner, last, ds in blocks(arch):
        cur = h
        for i in inner + [last]:
            cin, cout, k, s = geo(i)
            ho = (cur + 2 * (k // 2) - k) // s + 1
            out[i] = (cin, cout, k, s, cur, ho, i == last)
            cur = ho
        if ds is not None:
            cin, cout, k, s = geo(ds)
            out[ds] = (cin, cout, k, s, h, (h - 1) // s + 1, False)
        h = cur
    return tuple(out)


@functools.lru_cache(maxsize=None)
def blocks(arch: str = 'resnet50') -> Tuple[Tuple[List[int], int, Optional[int]], ...]:
    """Per residual block: (the indices of its inner convs, the index of the conv that adds the shortcut, the index of
    its downsample or None), in execution order."""
    out, cur = [], None
    for i, (ck, _) in enumerate(conv_keys(arch)):
        if i == 0:
            continue
        pre = '.'.join(ck.split('.')[:2])
        if cur is None or cur[0] != pre:
            cur = [pre, [], None, None]
            out.append(cur)
        if 'downsample' in ck:
            cur[3] = i
        else:
            cur[1].append(i)
    return tuple((c[1][:-1], c[1][-1], c[3]) for c in out)


def fold(sd, index: int, arch: str = 'resnet50') -> Tuple[torch.Tensor, torch.Tensor]:
    """Conv ``index`` of the plan with BN folded in float64: (W (N, K) in the GEMM's k order, bias); the stem keeps the
    OIHW order (c, ky, kx), the others (ky, kx, c)."""
    sd = strip_prefix(sd, RESNET_PREFIX)
    ck, bk = conv_keys(arch)[index]
    w, b = fold_bn(sd, bk, sd[ck + '.weight'])
    if index == 0:
        return w.reshape(w.shape[0], -1), b
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1), b


def stem(sd, x: torch.Tensor, arch: str = 'resnet50') -> Pair:
    """7x7/s2 conv + BN + ReLU of the NCHW image -> (B*3600, 64) rows (fp32 CUDA-core stage)."""
    w, b = fold(sd, 0, arch)
    cols = F.unfold(x.double(), 7, padding=3, stride=2).transpose(1, 2).reshape(-1, w.shape[1])
    return gemm64.simt(cols, w, b, True)


maxpool = gemm64.resnet_maxpool
avgpool = gemm64.avgpool


def conv(sd, index: int, x: torch.Tensor, batch: int, residual: Optional[torch.Tensor] = None,
         arch: str = 'resnet50') -> Pair:
    """Conv ``index`` + BN (+ the shortcut) (+ ReLU, all but a downsample) on input rows ``x`` (B*H*W, C)."""
    cin, _, ksize, stride, hin, _, _ = stage_table(arch)[index]
    w, b = fold(sd, index, arch)
    a = gemm64.patches(x.reshape(batch, hin, hin, cin), ksize, stride, ksize // 2)
    return gemm64.gemm(a, w, b, 'downsample' not in conv_keys(arch)[index][0], residual=residual)


def heads(sd, pooled: torch.Tensor) -> Pair:
    """fc_ori | fc_shape | fc_exp | fc_tex on the pooled features -> (B, 102) (tensor-core stage, no activation)."""
    return gemm64.gemm(pooled, *linear_heads(strip_prefix(sd, RESNET_PREFIX), HEADS), False)


@torch.no_grad()
def forward64(sd, x: torch.Tensor, arch: str = 'resnet50') -> Tuple[torch.Tensor, torch.Tensor]:
    """The whole network as the chain of the oracle's stages, in float64, on crops ``x`` (B,3,120,120): (out102,
    pooled)."""
    b = x.shape[0]
    X = maxpool(stem(sd, x, arch)[0], b).double()
    for inner, last, ds in blocks(arch):
        cur = X
        for i in inner:
            cur = conv(sd, i, cur, b, arch=arch)[0]
        ident = conv(sd, ds, X, b, arch=arch)[0] if ds is not None else X
        X = conv(sd, last, cur, b, ident, arch=arch)[0]
    pooled = avgpool(X, b)[0]
    return heads(sd, pooled)[0], pooled


@torch.no_grad()
def resnet_forward(sd, x: torch.Tensor, arch: str = 'resnet50', prefix: str = RESNET_PREFIX):
    """ResNet._forward_impl of ``arch`` in the dtype of ``x`` with torch's own convs (resnet_backbone.py:50-249), the
    ``reference_port.resnet50_forward`` of every arch: (out102 = ori|shape|exp|tex, pooled feature)."""
    sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    table = stage_table(arch)

    def bn(t, key):
        return F.batch_norm(t, sd[key + '.running_mean'], sd[key + '.running_var'], sd[key + '.weight'], sd[key + '.bias'],
                            False, 0.0, BN_EPS)

    keys = conv_keys(arch)

    def cbn(t, i):
        ck, bk = keys[i]
        _, _, k, s, _, _, _ = table[i]
        return bn(F.conv2d(t, sd[ck + '.weight'], None, s, k // 2), bk)

    x = F.max_pool2d(F.relu(cbn(x, 0)), 3, 2, 1)                                       # :229-232
    for inner, last, ds in blocks(arch):
        out = x
        for i in inner:
            out = F.relu(cbn(out, i))
        identity = cbn(x, ds) if ds is not None else x
        x = F.relu(cbn(out, last) + identity)
    pooled = torch.flatten(F.adaptive_avg_pool2d(x, 1), 1)                             # :239-240
    heads_ = [F.linear(pooled, sd[f'{k}.weight'], sd[f'{k}.bias']) for k in ('fc_ori', 'fc_shape', 'fc_exp', 'fc_tex')]
    return torch.cat(heads_, 1), pooled                                                # :242-246


# ---- batches and faces: those of gemm64 -- every arch has the four ResNet-50 map sizes (900 / 225 / 64 / 16) ------------
MAPS = gemm64.RESNET_MAPS
BATCHES = gemm64.RESNET_BATCHES
faces = gemm64.resnet_faces
