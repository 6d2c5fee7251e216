"""Float64 per-stage oracle of the GhostNet backbone, with a per-element error scale.  TEST INFRASTRUCTURE.

The contract is that of ``gemm64.py``: every stage is fed the exact fp32 tensors the GPU stage was fed (normally the GPU's
own outputs of earlier stages) and returns ``(want, S)``; a stage passes when |got - want| <= tau * S at every element.
BatchNorm is folded here, in float64, from the state dict (``check64.fold_bn``).

  * the 1x1 convs, the SE FCs, ConvBnAct, conv_head and the heads run on ``tc_gemm_kernel``: ``gemm64.gemm`` with the
    row scale taken from the true max |a| of each row.
  * the stem and the depthwise convs (the ghost modules' cheap operation, conv_dw, the shortcut's depthwise) run in
    fp32 on CUDA cores: S = sum_k |a_k||w_k| + |b|, plus |x1| + |residual| where the ghost pass adds the shortcut.
  * the pools: ``gemm64.avgpool``.  The SE gate x * relu6(z + 3) / 6: S = |x| (|z| + 3) / 6.

Block 3's conv_reduce has 20 output channels; the library pads it to 24 with zero weight rows and biases (and its
conv_expand to K = 24 with zero columns), so that stage has 24 columns here too, the last four exactly 0.

Stage numbering is that of ``syn_debug_ghost_until``: one stage per launch output, in launch order (``stage_table``).
Rows are what the GPU stores: one per NHWC pixel, or one per face for the SE vectors and after the final pool.
"""
from __future__ import annotations

import functools
import math
from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from oracle import gemm64
from oracle.check64 import Pair, fold_bn, linear_heads

HEADS = ('classifier_ori', 'classifier_shape', 'classifier_exp', 'classifier_texture')


# The bar: |got - want| <= TAU[kind] * S at every element, per stage kind (``kind``), at most 4x the worst ratio measured
# on an H100 80GB HBM3 (132 SMs, 700 W power limit) over the batches and both checkpoints of tests/test_gpu_ghostnet.py
# (worst in the comment).  The SE pools sum up to 225 pixels per channel, so their ratio is ~10x that of the final
# 16-pixel pool.
TAU = {'gemm': 5.3e-6,      # 1.33e-06: ghost2's primary GEMM of block 15 (K = 960) at B = 129
       'dw': 1.4e-6,        # 4.31e-07: the stem at B = 128; the depthwise and ghost passes alone 2.47e-07
       'pool': 8.5e-6,      # 2.13e-06: block 4's SE pool (225 pixels summed in fp32) at B = 128
       'gate': 5.8e-7}      # 1.47e-07: the SE gate of block 9 at B = 129
# Negative controls (test_negative_controls_fail_the_bar): bf16 weights measure 8.13e-04 on block 9's ghost2 primary GEMM
# and 2.17e-04 on block 10's conv_reduce (153x and 41x the gemm bar), rowmax_in / 8 1.11e-01 and 1.87e-02.

# The rescaled checkpoint of the tests (synth_ghost.reparametrize_ghostnet): hidden-channel factors 2^lo .. 2^hi.
WIDE = dict(seed=11, lo=-6, hi=4)


def over(ratios):
    """The stages of a ``stage_check.Ratios`` above their kind's bar in TAU."""
    return {s: v for s, v in ratios.items() if v[0] > TAU[v[2]]}


def pad8(n: int) -> int:
    return -(-n // 8) * 8


@functools.lru_cache(maxsize=None)
def blocks() -> Tuple[dict, ...]:
    """One dict per GhostBottleneck of ghostnet() at width 1.0: channels, kernel, stride, SE width, map sizes, key
    prefix -- from the reference's cfgs (ghostnet_backbone.py:243-266) and PyTorch's conv arithmetic."""
    from synergynet_b200.backbone import GHOSTNET_CFGS, _make_divisible
    out, cin, h = [], 16, 60
    for i, cfg in enumerate(GHOSTNET_CFGS):
        for j, (k, exp, c, se, s) in enumerate(cfg):
            mid, cout = _make_divisible(exp, 4), _make_divisible(c, 4)
            ho = (h + 2 * (k // 2) - k) // s + 1
            out.append(dict(cin=cin, mid=mid, cout=cout, k=k, s=s, red=_make_divisible(mid * se, 4) if se else 0,
                            h=h, ho=ho, p=f'blocks.{i}.{j}.', short=not (cin == cout and s == 1)))
            cin, h = cout, ho
    return tuple(out)


@functools.lru_cache(maxsize=None)
def stage_table() -> Tuple[dict, ...]:
    """The stages in launch order: op, block index (or None), rows per face, columns, whether it records row maxima,
    and the stages whose outputs it reads (-1: the crops)."""
    t = []

    def add(op, b, rows, cols, rm, inputs):
        t.append(dict(op=op, block=b, rows=rows, cols=cols, rowmax=rm, inputs=tuple(inputs)))
        return len(t) - 1

    x = add('stem', None, 3600, 16, True, (-1,))
    for bi, b in enumerate(blocks()):
        P, PO = b['h'] ** 2, b['ho'] ** 2
        x1 = add('primary1', bi, P, b['mid'] // 2, False, (x,))
        m = add('ghost1', bi, P, b['mid'], True, (x1,))
        if b['s'] > 1:
            m = add('dw', bi, PO, b['mid'], True, (m,))
        if b['red']:
            q = add('se_pool', bi, 1, b['mid'], True, (m,))
            z1 = add('se_reduce', bi, 1, pad8(b['red']), True, (q,))
            z2 = add('se_expand', bi, 1, b['mid'], False, (z1,))
            m = add('se_apply', bi, PO, b['mid'], True, (m, z2))
        x2 = add('primary2', bi, PO, b['cout'] // 2, False, (m,))
        r = x
        if b['short']:
            d = add('sc_dw', bi, PO, b['cin'], True, (x,))
            r = add('sc_pw', bi, PO, b['cout'], False, (d,))
        x = add('ghost2', bi, PO, b['cout'], True, (x2, r))
    c = add('conv_bn_act', None, 16, 960, False, (x,))
    q = add('pool', None, 1, 960, True, (c,))
    f = add('conv_head', None, 1, 1280, True, (q,))
    add('heads', None, 1, 102, False, (f,))
    return tuple(t)


NUM_STAGES = len(stage_table())


def kind(op: str) -> str:
    """The bar a stage is held to: 'gemm' (tensor cores), 'dw' (fp32 CUDA-core convs), 'pool', 'gate'."""
    if op in ('stem', 'ghost1', 'ghost2', 'dw', 'sc_dw'):
        return 'dw'
    if op in ('se_pool', 'pool'):
        return 'pool'
    return 'gate' if op == 'se_apply' else 'gemm'


def _bn(sd, conv: str, bn: str) -> Tuple[torch.Tensor, torch.Tensor]:
    return fold_bn(sd, bn, sd[conv + '.weight'])


def _nchw(rows: torch.Tensor, nf: int) -> torch.Tensor:
    hw = int(round(math.sqrt(rows.shape[0] // nf)))
    return rows.double().view(nf, hw, hw, rows.shape[1]).permute(0, 3, 1, 2)


def _rows(x: torch.Tensor) -> torch.Tensor:
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])


def _depthwise(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, stride: int, nf: int) -> Pair:
    a = _nchw(x, nf)
    c, k = a.shape[1], w.shape[-1]
    y = F.conv2d(a, w, None, stride, k // 2, 1, c) + b.view(1, -1, 1, 1)
    s = F.conv2d(a.abs(), w.abs(), None, stride, k // 2, 1, c) + b.abs().view(1, -1, 1, 1)
    return _rows(y), _rows(s)


def _w2(w: torch.Tensor) -> torch.Tensor:
    return w.reshape(w.shape[0], -1)


def se_weights(sd, b: dict) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """conv_reduce (N padded to a multiple of 8 with zero rows and biases) and conv_expand (K padded the same way with
    zero columns), as the library builds them: (w_reduce, b_reduce, w_expand, b_expand), float64."""
    p = b['p'] + 'se.'
    wr, br = _w2(sd[p + 'conv_reduce.weight']).double(), sd[p + 'conv_reduce.bias'].double()
    we, be = _w2(sd[p + 'conv_expand.weight']).double(), sd[p + 'conv_expand.bias'].double()
    n = pad8(wr.shape[0])
    wr = torch.cat([wr, wr.new_zeros(n - wr.shape[0], wr.shape[1])])
    br = torch.cat([br, br.new_zeros(n - br.shape[0])])
    we = torch.cat([we, we.new_zeros(we.shape[0], n - we.shape[1])], dim=1)
    return wr, br, we, be


def gate(x: torch.Tensor, z: torch.Tensor, nf: int) -> Pair:
    """x * relu6(z + 3) / 6 with z (B, C) broadcast over each face's rows of x (B*P, C)."""
    x = x.double().view(nf, -1, x.shape[1])
    z = z.double().view(nf, 1, -1)
    y = x * (z + 3.0).clamp(0.0, 6.0) / 6.0
    s = x.abs() * (z.abs() + 3.0) / 6.0
    return y.reshape(-1, y.shape[2]), s.reshape(-1, s.shape[2])


def stage(sd, s: int, outs: Dict[int, torch.Tensor], nf: int) -> Pair:
    """Stage ``s`` of syn_debug_ghost_until on the outputs of the stages it reads: ``outs[i]`` is stage i's output
    (rows as the GPU stores them), ``outs[-1]`` the NCHW crops; ``nf`` faces."""
    st = stage_table()[s]
    op, inp = st['op'], [outs[i] for i in st['inputs']]
    b = blocks()[st['block']] if st['block'] is not None else None
    if op == 'stem':
        w, bias = _bn(sd, 'conv_stem', 'bn1')
        cols = F.unfold(inp[0].double(), 3, padding=1, stride=2).transpose(1, 2).reshape(-1, 27)
        return gemm64.simt(cols, _w2(w), bias, True)
    if op in ('primary1', 'primary2'):
        g = b['p'] + ('ghost1' if op == 'primary1' else 'ghost2')
        w, bias = _bn(sd, g + '.primary_conv.0', g + '.primary_conv.1')
        return gemm64.gemm(inp[0], _w2(w), bias, op == 'primary1')
    if op in ('ghost1', 'ghost2'):
        g = b['p'] + op
        relu = op == 'ghost1'
        w, bias = _bn(sd, g + '.cheap_operation.0', g + '.cheap_operation.1')
        x1 = inp[0].double()
        y, sy = _depthwise(inp[0], w, bias, 1, nf)
        if relu:
            y = y.clamp_min(0.0)
        lo, slo = x1, x1.abs()
        if op == 'ghost2':
            r = inp[1].double()
            c = x1.shape[1]
            lo, slo = x1 + r[:, :c], slo + r[:, :c].abs()
            y, sy = y + r[:, c:], sy + r[:, c:].abs()
        return torch.cat([lo, y], dim=1), torch.cat([slo, sy], dim=1)
    if op == 'dw':
        w, bias = _bn(sd, b['p'] + 'conv_dw', b['p'] + 'bn_dw')
        return _depthwise(inp[0], w, bias, b['s'], nf)
    if op == 'sc_dw':
        w, bias = _bn(sd, b['p'] + 'shortcut.0', b['p'] + 'shortcut.1')
        return _depthwise(inp[0], w, bias, b['s'], nf)
    if op == 'sc_pw':
        w, bias = _bn(sd, b['p'] + 'shortcut.2', b['p'] + 'shortcut.3')
        return gemm64.gemm(inp[0], _w2(w), bias, False)
    if op in ('se_pool', 'pool'):
        return gemm64.avgpool(inp[0], nf)
    if op == 'se_reduce':
        wr, br, _, _ = se_weights(sd, b)
        return gemm64.gemm(inp[0], wr, br, True)
    if op == 'se_expand':
        _, _, we, be = se_weights(sd, b)
        return gemm64.gemm(inp[0], we, be, False)
    if op == 'se_apply':
        return gate(inp[0], inp[1], nf)
    if op == 'conv_bn_act':
        w, bias = _bn(sd, 'blocks.9.0.conv', 'blocks.9.0.bn1')
        return gemm64.gemm(inp[0], _w2(w), bias, True)
    if op == 'conv_head':
        return gemm64.gemm(inp[0], _w2(sd['conv_head.weight']), sd['conv_head.bias'], True)
    return gemm64.gemm(inp[0], *linear_heads(sd, HEADS), False)


@torch.no_grad()
def forward64(sd, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The whole network in float64 on crops ``x`` (B,3,120,120): (out102, feat1280), what GhostNet.forward computes
    (out102) and the conv_head output after its ReLU."""
    outs = {-1: x.double()}
    for s in range(NUM_STAGES):
        outs[s] = stage(sd, s, outs, x.shape[0])[0]
    return outs[NUM_STAGES - 1], outs[NUM_STAGES - 2]


# ---- batches and faces that put the tile edges under a check ----------------------------------------------------------

MAPS = (3600, 900, 225, 64, 16, 1)       # rows per face of the GEMMs: the five map sizes, and the SE / head vectors
BATCHES = (2, 33, 128, 129)


def dw_rows(ho: int) -> int:
    """Output rows per CTA of dw_kernel (csrc/mbv1_host.inl dw_band): about 128 pixels."""
    return min(ho, -(-128 // ho))


def last_tile_kinds(p: int, batches) -> set:
    """Shapes of the GEMM's last 128-row tile over the batches at p rows per face: 'min' (the fewest rows a ragged tile
    can hold there, gcd(p, 128)), 'full' (128 rows) and 'mid' (anything in between)."""
    g = math.gcd(p, gemm64.TILE)
    kinds = set()
    for b in batches:
        r = b * p % gemm64.TILE
        kinds.add('full' if r == 0 else 'min' if r == g else 'mid')
    return kinds


def check_ghost_batches(batches=BATCHES) -> None:
    """At every map size, and for the per-face rows of the SE and head GEMMs, the batches put the GEMM's last 128-row tile
    at its fewest rows, at 128 rows and in between (where the size allows a value in between); and they run the
    depthwise kernel's last partial band on the last face of each batch, which the checked faces include."""
    for p in MAPS:
        g = math.gcd(p, gemm64.TILE)
        need = {'min', 'full'} | ({'mid'} if gemm64.TILE // g > 2 else set())
        kinds = last_tile_kinds(p, batches)
        assert need <= kinds, (p, kinds)
    assert [ho for ho in (60, 30, 15, 8, 4) if ho % dw_rows(ho)], 'no map size has a partial depthwise band'
    assert batches and all(b - 1 in faces(b) for b in batches), 'no batch runs a last partial band under the check'


def faces(batch: int) -> list:
    """``gemm64.tile_edge_faces`` over the GhostNet row counts per face."""
    return gemm64.tile_edge_faces(batch, MAPS)
