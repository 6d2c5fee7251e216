"""A seeded, calibrated GhostNet checkpoint in the reference's key schema, and an exact reparametrisation of it that
spreads the hidden-channel magnitudes.  TEST INFRASTRUCTURE.

As ``synth_mbv1`` does for MobileNetV1, every BatchNorm gets the float64 batch statistics of its own input on a small
calibration batch, perturbed, and randomised affine parameters, so that the signal survives all 16 bottlenecks like in
a trained checkpoint.  The SE convs get non-zero biases, and each conv_expand is scaled so that its gate logits spread
over about +-9 on the calibration batch: the hard-sigmoid's clamps at -3 and +3 are both exercised.  Keys have no
prefix, as ``ghostnet_backbone.ghostnet().state_dict()`` returns them.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle.synth_model import _pow2_factors
from synergynet_b200 import synthetic

_CACHE: Dict[int, Dict[str, torch.Tensor]] = {}
EPS = 1e-5


@torch.no_grad()
def build_ghostnet_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    if seed in _CACHE:
        return _CACHE[seed]
    from synergynet_b200 import backbone
    from oracle import ghost64
    m = backbone.ghostnet()
    synthetic.seeded_init_(m, 700 + seed)
    synthetic.randomize_batchnorm_(m, 700 + seed)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(7000 + seed)
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(8, seed=300 + seed)).double()

    def conv(t, key, stride=1, groups=1, bias=False):
        w = sd[key + '.weight'].double()
        return F.conv2d(t, w, sd[key + '.bias'].double() if bias else None, stride, w.shape[-1] // 2, 1, groups)

    def bn(y, key, relu):
        mean, var = y.mean(dim=(0, 2, 3)), y.var(dim=(0, 2, 3), unbiased=False)
        c = mean.numel()
        mean = mean + 0.1 * var.sqrt() * torch.randn(c, generator=g, dtype=torch.float64)
        var = var * (0.8 + 0.4 * torch.rand(c, generator=g, dtype=torch.float64)) + 1e-6
        sd[key + '.running_mean'], sd[key + '.running_var'] = mean.float(), var.float()
        p = lambda k: sd[f'{key}.{k}'].double().view(1, -1, 1, 1)
        y = (y - p('running_mean')) / torch.sqrt(p('running_var') + EPS) * p('weight') + p('bias')
        return y.clamp_min(0.0) if relu else y

    def ghost(t, key, relu):
        x1 = bn(conv(t, key + '.primary_conv.0'), key + '.primary_conv.1', relu)
        x2 = bn(conv(x1, key + '.cheap_operation.0', groups=x1.shape[1]), key + '.cheap_operation.1', relu)
        return torch.cat([x1, x2], dim=1)

    x = bn(conv(x, 'conv_stem', 2), 'bn1', True)
    for b in ghost64.blocks():
        p = b['p']
        y = ghost(x, p + 'ghost1', True)
        if b['s'] > 1:
            y = bn(conv(y, p + 'conv_dw', b['s'], b['mid']), p + 'bn_dw', False)
        if b['red']:
            sd[p + 'se.conv_reduce.bias'] = 0.1 * torch.randn(b['red'], generator=g)
            z1 = conv(y.mean(dim=(2, 3), keepdim=True), p + 'se.conv_reduce', bias=True).clamp_min(0.0)
            z0 = conv(z1, p + 'se.conv_expand')
            sd[p + 'se.conv_expand.weight'] = (sd[p + 'se.conv_expand.weight'].double() * 5.0 / z0.std()).float()
            sd[p + 'se.conv_expand.bias'] = torch.randn(b['mid'], generator=g)
            z = conv(z1, p + 'se.conv_expand', bias=True)
            y = y * (z + 3.0).clamp(0.0, 6.0) / 6.0
        y = ghost(y, p + 'ghost2', False)
        if b['short']:
            r = bn(conv(x, p + 'shortcut.0', b['s'], b['cin']), p + 'shortcut.1', False)
            r = bn(conv(r, p + 'shortcut.2'), p + 'shortcut.3', False)
        else:
            r = x
        x = y + r
    bn(conv(x, 'blocks.9.0.conv'), 'blocks.9.0.bn1', True)
    _CACHE[seed] = sd
    return sd


@torch.no_grad()
def reparametrize_ghostnet(sd: Dict[str, torch.Tensor], seed: int, lo: int, hi: int) -> Dict[str, torch.Tensor]:
    """The same network with every bottleneck's hidden (mid) channels spread over 2^lo .. 2^hi: the gamma and beta of
    ghost1's two BatchNorms (and of bn_dw) are multiplied by per-channel factors 2^k and the consumers divide by the
    same factors -- the cheap operation's channel after primary_conv, conv_dw's channel, conv_reduce's and ghost2
    primary_conv's input columns.  ReLU(f x) = f ReLU(x) for f > 0, the depthwise convs and the pool are per channel
    and linear, and the SE gate, computed from the rescaled conv_reduce, is unchanged; powers of two make this exact in
    fp32, so the output is unchanged while every row maximum the GEMMs scale by moves."""
    from oracle import ghost64
    out = {k: v.clone() for k, v in sd.items()}
    g = torch.Generator().manual_seed(seed)

    def scale_bn(key):
        f = _pow2_factors(out[key + '.weight'].numel(), g, lo, hi)
        out[key + '.weight'] *= f
        out[key + '.bias'] *= f
        return f

    for b in ghost64.blocks():
        p = b['p']
        f1 = scale_bn(p + 'ghost1.primary_conv.1')
        out[p + 'ghost1.cheap_operation.0.weight'] /= f1.view(-1, 1, 1, 1)
        f = torch.cat([f1, scale_bn(p + 'ghost1.cheap_operation.1')])
        if b['s'] > 1:
            out[p + 'conv_dw.weight'] /= f.view(-1, 1, 1, 1)
            f = scale_bn(p + 'bn_dw')
        if b['red']:
            out[p + 'se.conv_reduce.weight'] /= f.view(1, -1, 1, 1)
        out[p + 'ghost2.primary_conv.0.weight'] /= f.view(1, -1, 1, 1)
    return out
