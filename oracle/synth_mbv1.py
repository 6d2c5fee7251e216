"""Seeded, calibrated MobileNetV1 checkpoints in the reference's key schema, and an exact reparametrisation of them that
spreads the hidden-channel magnitudes.  TEST INFRASTRUCTURE.

The reference initialises every BatchNorm to the identity (mobilenetv1_backbone.py:100-106), which would leave BN folding
untested, and with arbitrary statistics a random MobileNetV1 forgets its input after a few depthwise convs (each one
shrinks the signal by about sqrt(2 / C)).  So, as ``synth_model.build_state_dict`` does for MobileNetV2, each BatchNorm
gets the float64 batch statistics of its own input on a small calibration batch, perturbed, and randomised affine
parameters: the signal survives all 27 convolutions like in a trained checkpoint.  Keys have no prefix, as
``mobilenetv1_backbone.mobilenet_*().state_dict()`` returns them.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle.synth_model import _pow2_factors
from synergynet_b200 import synthetic

_CACHE: Dict[tuple, Dict[str, torch.Tensor]] = {}


@torch.no_grad()
def build_mobilenet_v1_state_dict(seed: int = 0, arch: str = 'mobilenet_1') -> Dict[str, torch.Tensor]:
    key = (arch, seed)
    if key in _CACHE:
        return _CACHE[key]
    from synergynet_b200 import backbone
    from synergynet_b200.backbone import mobilenet_v1_conv_keys
    from oracle import mbv1_64
    m = getattr(backbone, arch)()
    synthetic.seeded_init_(m, 600 + seed)
    synthetic.randomize_batchnorm_(m, 600 + seed)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(6000 + seed)
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(8, seed=200 + seed)).double()
    table = mbv1_64.stage_table(arch)
    for (ck, bk), (_, cout, _, stride, groups, _, _) in zip(mobilenet_v1_conv_keys(), table):
        y = F.conv2d(x, sd[ck + '.weight'].double(), None, stride, 1 if groups > 1 or ck == 'conv1' else 0, 1, groups)
        mean, var = y.mean(dim=(0, 2, 3)), y.var(dim=(0, 2, 3), unbiased=False)
        mean = mean + 0.1 * var.sqrt() * torch.randn(cout, generator=g, dtype=torch.float64)
        var = var * (0.8 + 0.4 * torch.rand(cout, generator=g, dtype=torch.float64)) + 1e-6
        sd[bk + '.running_mean'] = mean.float()
        sd[bk + '.running_var'] = var.float()
        p = lambda k: sd[f'{bk}.{k}'].double().view(1, -1, 1, 1)
        x = ((y - p('running_mean')) / torch.sqrt(p('running_var') + 1e-5) * p('weight') + p('bias')).clamp_min(0.0)
    _CACHE[key] = sd
    return sd


@torch.no_grad()
def reparametrize_mobilenet_v1(sd: Dict[str, torch.Tensor], seed: int, lo: int, hi: int) -> Dict[str, torch.Tensor]:
    """The same network with hidden channels spread over 2^lo .. 2^hi, in the manner of ``reparametrize_resnet``: every
    BatchNorm's gamma and beta are multiplied by per-channel factors 2^k and the consumer of those channels divides by
    the same factors -- conv_sep's input columns after bn_dw, the next conv_dw's channel after bn1 / bn_sep, and the
    four heads' input columns after the last bn_sep (the average pool is linear).  Every BN is followed by a ReLU, and
    ReLU(f x) = f ReLU(x) for f > 0; powers of two make this exact in fp32, so the output is unchanged while every row
    maximum the GEMMs scale by moves."""
    from synergynet_b200.backbone import mobilenet_v1_conv_keys
    out = {k: v.clone() for k, v in sd.items()}
    g = torch.Generator().manual_seed(seed)
    keys = mobilenet_v1_conv_keys()
    for i, (_, bk) in enumerate(keys):
        f = _pow2_factors(out[bk + '.weight'].numel(), g, lo, hi)
        out[bk + '.weight'] *= f
        out[bk + '.bias'] *= f
        if i + 1 < len(keys):
            w = out[keys[i + 1][0] + '.weight']
            if i % 2 == 1:                                   # bn_dw -> conv_sep: input columns
                w /= f.view(1, -1, 1, 1)
            else:                                            # bn1 / bn_sep -> the next conv_dw: one channel each
                w /= f.view(-1, 1, 1, 1)
        else:
            for h in ('fc_ori', 'fc_shape', 'fc_exp', 'fc_tex'):
                out[h + '.weight'] /= f.view(1, -1)
    return out
