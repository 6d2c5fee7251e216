"""Seeded checkpoints of the seven ResNet backbones in the reference's key schema, and an exact reparametrisation of them
that spreads the hidden-channel magnitudes.  TEST INFRASTRUCTURE.

``build_resnet_state_dict(seed, 'resnet50')`` is ``synth_model.build_resnet50_state_dict(seed)`` bit for bit (the golden
vectors of resnet50 depend on it), and ``reparametrize_resnet(sd, 'resnet50', ...)`` is
``synth_model.reparametrize_resnet``: the other arches get the same treatment.
"""
from __future__ import annotations

from typing import Dict

import torch

from oracle.synth_model import _pow2_factors, _rescale_hidden
from synergynet_b200 import synthetic

_CACHE: Dict[tuple, Dict[str, torch.Tensor]] = {}


@torch.no_grad()
def build_resnet_state_dict(seed: int = 0, arch: str = 'resnet50') -> Dict[str, torch.Tensor]:
    """Seeded state dict of ``resnet_backbone.<arch>()`` (keys without prefix): kaiming convs like the reference's own
    init, randomised BatchNorm affine parameters and running statistics so that BN folding is exercised.  ReLU networks
    with residual connections keep their signal without calibration, but every block adds its branch to the stream, so
    magnitudes grow with the number of blocks: ResNet-50's 16 blocks end at a few hundred, ResNet-152's 50 at ~1e9.  The
    last BatchNorm of every block (gamma and beta) is therefore scaled by 16 / the number of blocks -- 1 for resnet50,
    34 and wide_resnet50_2, 2 for resnet18, 16/33 and 16/50 for the deeper ones -- which keeps out102 at 10 .. 200 for
    every arch."""
    key = (arch, seed)
    if key in _CACHE:
        return _CACHE[key]
    from synergynet_b200 import backbone
    m = getattr(backbone, arch)()
    synthetic.seeded_init_(m, 300 + seed)
    synthetic.randomize_batchnorm_(m, 300 + seed)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    from oracle import resnets64
    blocks, keys = resnets64.blocks(arch), resnets64.conv_keys(arch)
    if len(blocks) != 16:
        for _, last, _ in blocks:
            bk = keys[last][1]
            sd[bk + '.weight'] *= 16 / len(blocks)
            sd[bk + '.bias'] *= 16 / len(blocks)
    _CACHE[key] = sd
    return sd


@torch.no_grad()
def reparametrize_resnet(sd: Dict[str, torch.Tensor], arch: str, seed: int, lo: int, hi: int,
                         prefix: str = '') -> Dict[str, torch.Tensor]:
    """``arch`` with a wide spread of hidden-channel magnitudes: in every block, the BatchNorm after each inner conv
    (bn1, and bn2 of a Bottleneck) has its channels scaled by powers of two 2^k, k in [lo, hi], and the next conv's
    input columns divided by the same factors.  Powers of two make this exact in fp32: the hidden activations become
    exactly f * the original, and every block output is unchanged."""
    from oracle import resnets64
    keys = resnets64.conv_keys(arch)
    out = {k: v.clone() for k, v in sd.items()}
    g = torch.Generator().manual_seed(seed)
    for inner, last, _ in resnets64.blocks(arch):
        chain = list(inner) + [last]
        for a, b in zip(chain[:-1], chain[1:]):
            bn = prefix + keys[a][1]
            f = _pow2_factors(out[bn + '.weight'].numel(), g, lo, hi)
            _rescale_hidden(out, bn, [(prefix + keys[b][0] + '.weight', 0)], f)
    return out
