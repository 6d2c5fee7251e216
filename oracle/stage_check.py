"""The per-stage bar of the backbone engines against the float64 oracle (``block64``).  TEST INFRASTRUCTURE.

Each stage is fed the GPU's own output of the previous stage, so errors do not accumulate and every element of every
stage is held to |got - want| <= TAU * S, S being the stage's first-order error scale.  The unfused engines are checked
conv by conv (52 convs), the fused engine block by block (17 blocks, conv index 3b - 1); then the pooled feature and
the 62 params.  Shared by every GPU test that holds a backbone engine to that bar.
"""
from __future__ import annotations

import types
from typing import Dict, List, Tuple

import torch

from oracle import block64
from synergynet_b200 import _lib
from synergynet_b200.backbone import conv_plan

# The bar: |got - want| <= TAU * S at every element.  S is a first-order bound, and a bound carried through the three
# convs of a fused block is far more pessimistic than the bound of one conv (it adds |W| * S of every hidden element,
# while real rounding errors cancel), so one TAU for both would leave the fused blocks ~40x of slack.  TAU is therefore
# set per engine and stage kind, at most 4x the worst ratio measured on an H100 80GB HBM3 (132 SMs, 700 W power limit)
# over the three batches of tests/test_gpu_blocks.py and the rescaled checkpoint (worst in the comment):
TAU = {
    'simt_fp32': {'conv': 1.3e-6,        # 3.29e-07 (conv 6)
                  'pool': 8e-7,          # 2.10e-07
                  'params': 8e-8},       # 2.00e-08
    'tc_bf16x3': {'conv': 4.9e-6,        # 1.24e-06 (conv 44, rescaled checkpoint; 1.235e-06 on the original)
                  'pool': 9e-7,          # 2.38e-07
                  'params': 9e-8},       # 2.27e-08
    'tc_fused': {'block': 1.4e-7,        # 3.54e-08 (block 2)
                 'pool': 6.9e-7,         # 1.75e-07 (tail kernel)
                 'params': 8.8e-8},      # 2.22e-08
}
# The single-pass engine measures 2.06e-06 (block 15) to 3.40e-05 (block 1) and 2.46e-05 at the tail: >= 14x the bar.
ENGINES = {'simt_fp32': _lib.ENGINE_SIMT_FP32, 'tc_bf16x3': _lib.ENGINE_TC_BF16X3, 'tc_fused': _lib.ENGINE_TC_FUSED}

Ratios = Dict[str, Tuple[float, tuple]]


def make_model(sd):
    from synergynet_b200 import model_building
    args = types.SimpleNamespace(arch='mobilenet_v2', img_size=120, devices_id=[0])
    m = model_building.SynergyNet(args)
    m.load_state_dict(sd, strict=True)
    m.eval()
    return m


def stage_ratios(eng, fused: bool, sd, x: torch.Tensor, faces: List[int]) -> Ratios:
    """{stage: (worst |got - want| / S, (face, y, x, channel))} over the given faces of batch ``x`` (on the GPU)."""
    fidx = torch.tensor(faces, device='cuda')
    pick = lambda t: t.index_select(0, fidx).cpu().double()
    img = pick(x)
    out = {}
    if fused:
        prev = img
        for b in range(1, 18):
            got = pick(eng.debug_forward_until(x, 3 * b - 1))
            out[f'block{b}'] = block64.worst(got, *block64.block(sd, b, prev))
            prev = got
        pool_want = block64.tail(sd, prev)
    else:
        got = {}
        for spec in conv_plan():
            got[spec.index] = pick(eng.debug_forward_until(x, spec.index))
            src = img if spec.index == 0 else got[spec.index - 1]
            skip = got[spec.index - 3] if spec.residual else None        # the block input, before its expand
            out[f'conv{spec.index}'] = block64.worst(got[spec.index], *block64.conv(sd, spec.index, src, skip))
        pool_want = block64.avgpool(got[len(got) - 1])
    params, pool = eng.forward(x, want_pool=True)
    pool = pick(pool)
    out['pool'] = block64.worst(pool, *pool_want)
    out['params'] = block64.worst(pick(params), *block64.heads(sd, pool))
    assert eng.poll_error() == 0
    assert eng.poll_saturation(warn=False) == 0
    return out


def tau(engine: str, stage: str) -> float:
    return TAU[engine][stage.rstrip('0123456789')]


def over(engine: str, ratios: Ratios) -> Ratios:
    """The stages of ``ratios`` above the bar."""
    return {k: v for k, v in ratios.items() if v[0] > tau(engine, k)}


def report(tag: str, ratios: Ratios) -> None:
    name, (r, where) = max(ratios.items(), key=lambda kv: kv[1][0])
    print(f'\n[{tag}] worst {r:.3e} at {name} {where}')
    print('  ' + '  '.join(f'{k}={v[0]:.2e}' for k, v in ratios.items()))
