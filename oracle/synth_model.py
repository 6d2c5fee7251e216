"""Seeded, *calibrated* synthetic checkpoint in the reference's key schema.  TEST INFRASTRUCTURE.

A randomly initialised MobileNetV2 in eval mode with arbitrary BatchNorm statistics forgets its
input after a few depthwise layers (kaiming fan_out weights shrink the signal by ~C/2 per
depthwise conv), so every crop would give the same 62 parameters and parity tests would only
exercise the bias path.  Here each BatchNorm's running statistics are set to the float64 batch
statistics of its own input on a small calibration batch (what training-mode BN would have
converged to), then perturbed, so that the signal survives all 52 convolutions like in a
trained checkpoint.  All randomness comes from seeded CPU generators; the statistics are computed
in float64 so that the fp32 result is reproducible across hosts.

Follows the module structure of reference backbone_nets/mobilenetv2_backbone.py:104-158.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from synergynet_b200 import synthetic
from synergynet_b200.backbone import conv_plan

_CACHE: Dict[int, Dict[str, torch.Tensor]] = {}


@torch.no_grad()
def build_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Full 445-key state dict (CPU fp32) of ``synergy3DMM.SynergyNet`` with synthetic 3DMM
    buffers (seed 0 model), seeded weights and calibrated BatchNorm statistics."""
    if seed in _CACHE:
        return _CACHE[seed]
    from synergynet_b200.params import ParamsPack, set_param_pack
    from synergynet_b200 import synergy3DMM
    pack = ParamsPack(arrays=synthetic.make_3dmm(seed=0))
    set_param_pack(pack)
    import contextlib, io
    with contextlib.redirect_stdout(io.StringIO()):
        model = synergy3DMM.SynergyNet()
    synthetic.seeded_init_(model, seed)
    synthetic.randomize_batchnorm_(model, seed)          # gamma/beta (and the PointNet BN stats)
    sd = model.state_dict()
    g = torch.Generator().manual_seed(5000 + seed)
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(8, seed=100 + seed)).double()
    pre = 'I2P.backbone.'
    block_in = None
    for spec in conv_plan():
        if spec.kind in ('expand', 'dw') and (spec.kind == 'expand' or spec.cin == 32 and spec.block == 1):
            block_in = x
        w = sd[pre + spec.conv_key + '.weight'].double()
        y = F.conv2d(x, w, None, spec.stride, (spec.ksize - 1) // 2, 1, spec.groups)
        mean = y.mean(dim=(0, 2, 3))
        var = y.var(dim=(0, 2, 3), unbiased=False)
        n = spec.cout
        mean = mean + 0.1 * var.sqrt() * torch.randn(n, generator=g, dtype=torch.float64)
        var = var * (0.8 + 0.4 * torch.rand(n, generator=g, dtype=torch.float64)) + 1e-6
        sd[pre + spec.bn_key + '.running_mean'].copy_(mean.float())
        sd[pre + spec.bn_key + '.running_var'].copy_(var.float())
        gamma = sd[pre + spec.bn_key + '.weight'].double()
        beta = sd[pre + spec.bn_key + '.bias'].double()
        rm = sd[pre + spec.bn_key + '.running_mean'].double()
        rv = sd[pre + spec.bn_key + '.running_var'].double()
        y = (y - rm.view(1, -1, 1, 1)) / torch.sqrt(rv.view(1, -1, 1, 1) + 1e-5) * gamma.view(1, -1, 1, 1) \
            + beta.view(1, -1, 1, 1)
        if spec.relu6:
            y = y.clamp(0, 6)
        if spec.residual:
            y = y + block_in
        x = y
    _calibrate_pointnet(sd, x.float().mean(dim=(2, 3)), seed)
    _CACHE[seed] = sd
    return sd


@torch.no_grad()
def reparametrize_streams(sd: Dict[str, torch.Tensor], seed: int, lo: int, hi: int) -> Dict[str, torch.Tensor]:
    """The same network with a wide spread of channel magnitudes, as trained checkpoints have.

    Only the block streams (the 16/24/32/64/96/160/320-channel tensors between blocks) can be rescaled without changing
    the function: they are the only tensors not followed by a ReLU6, which does not commute with scaling.  Channel c of
    each stream gets a factor f_c = 2^k with k an integer drawn from [lo, hi] (one channel at each end of the range):
    gamma and beta of every project BatchNorm that writes the stream are multiplied by f_c, and input column c of every
    conv that reads it (the expands of the following blocks and the last conv) is divided by f_c.  Powers of two make
    this exact in fp32: every block output becomes exactly f * the original and everything after it is unchanged."""
    out = {k: v.clone() for k, v in sd.items()}
    pre = 'I2P.backbone.'
    g = torch.Generator().manual_seed(seed)
    f = None
    for spec in conv_plan():
        if spec.kind in ('expand', 'last') and f is not None:
            out[pre + spec.conv_key + '.weight'] /= f.view(1, -1, 1, 1)
        if spec.kind == 'project':
            if not spec.residual:                              # first block of a stage: a new stream
                k = torch.randint(lo, hi + 1, (spec.cout,), generator=g)
                ends = torch.randperm(spec.cout, generator=g)[:2]
                k[ends[0]], k[ends[1]] = lo, hi
                f = torch.pow(2.0, k.double()).float()
            out[pre + spec.bn_key + '.weight'] *= f
            out[pre + spec.bn_key + '.bias'] *= f
    return out


STREAMS = (16, 24, 32, 64, 96, 160, 320)         # channels of the block streams, in network order


def stream_blocks(stream: int):
    """(blocks whose project conv writes the stream, blocks whose input it is; 18 stands for the tail, features.18)."""
    writers = [s.block for s in conv_plan() if s.kind == 'project' and s.cout == stream]
    readers = [s.block for s in conv_plan() if s.kind in ('expand', 'last') and s.cin == stream]
    assert writers and readers == [b + 1 for b in writers], (stream, writers, readers)
    return writers, readers


@torch.no_grad()
def scale_stream_channel(sd: Dict[str, torch.Tensor], stream: int, channel: int, factor: float) -> Dict[str, torch.Tensor]:
    """The same network with channel ``channel`` of one block stream multiplied by ``factor`` (> 0): gamma and beta of
    every project BatchNorm that writes the stream are multiplied by the fp32 factor, and input column ``channel`` of
    every conv that reads it (the following expands, or features.18 for the 320 stream) is divided by it -- the
    arithmetic of ``reparametrize_streams`` for one channel and any factor.  Exact in function; in fp32 only for a
    power of two, otherwise within the rounding of the rescaled weights."""
    out = {k: v.clone() for k, v in sd.items()}
    pre = 'I2P.backbone.'
    f = torch.tensor(factor, dtype=torch.float32)
    assert f > 0, factor
    for spec in conv_plan():
        if spec.kind == 'project' and spec.cout == stream:
            out[pre + spec.bn_key + '.weight'][channel] *= f
            out[pre + spec.bn_key + '.bias'][channel] *= f
        if spec.kind in ('expand', 'last') and spec.cin == stream:
            out[pre + spec.conv_key + '.weight'][:, channel] /= f
    return out


DEAD_INPUT_BOUND = 937.5         # the largest |x| the split-fp16 engines take unchanged (60000 / kActScale)


def _bn_scale(sd: Dict[str, torch.Tensor], bn: str) -> torch.Tensor:
    """gamma / sqrt(var + eps) of a BatchNorm in float64: what folding multiplies the conv weights by."""
    return sd[bn + '.weight'].double() / torch.sqrt(sd[bn + '.running_var'].double() + 1e-5)


@torch.no_grad()
def scale_hidden_channel(sd: Dict[str, torch.Tensor], block: int, channel: int, factor: float) -> Dict[str, torch.Tensor]:
    """Block ``block`` (1..17) with hidden channel ``channel`` dead and its folded expand weights ``factor`` times the
    rest's: the channel a trained checkpoint gets where BN folding divides by a near-zero running variance.  For block 1
    the hidden tensor is the stem's output, for the others the expand conv's.

    The conv weights of the channel are multiplied by ``factor`` and its BN beta set so that the folded bias is below
    -2 * sum |folded w| * 937.5: the pre-activation is negative for every input the split engines take, so the channel's
    hidden value is 0 after the ReLU6.  The input column of the block's project conv that reads the channel (through the
    depthwise conv) is set to 0, which changes nothing more in the function and keeps the dead channel's large error
    scale out of the project's.  This changes the function only through that one channel, which the original network
    had active; stream magnitudes stay as they were."""
    out = {k: v.clone() for k, v in sd.items()}
    pre = 'I2P.backbone.'
    plan = conv_plan()
    first = [s for s in plan if s.block == block and s.kind in ('expand', 'dw')][0]
    spec = plan[0] if first.kind == 'dw' else first                 # block 1: the stem is the expand
    proj = [s for s in plan if s.block == block and s.kind == 'project'][0]
    w = out[pre + spec.conv_key + '.weight']
    w[channel] *= torch.tensor(factor, dtype=torch.float32)
    bn = pre + spec.bn_key
    scale = _bn_scale(out, bn)[channel]
    reach = 2.0 * float((w[channel].double() * scale).abs().sum()) * DEAD_INPUT_BOUND
    # folded bias = beta - mean * scale
    out[bn + '.bias'][channel] = float(out[bn + '.running_mean'][channel].double() * scale) - reach
    out[pre + proj.conv_key + '.weight'][:, channel] = 0.0
    return out


@torch.no_grad()
def scale_output_channel(sd: Dict[str, torch.Tensor], conv_index: int, channel: int, factor: float,
                         bias: float = None) -> Dict[str, torch.Tensor]:
    """Output channel ``channel`` of conv ``conv_index`` with gamma and beta of its BN multiplied by ``factor``: its
    folded weights and bias scale by ``factor``, and, unlike ``scale_stream_channel``, the convs that read it are left
    as they are, so a tiny channel needs no reader column multiplied by up to 2^149.  Exact in fp32 for a power of two
    whose products stay normal.  ``factor`` 0 makes an all-zero channel; with ``bias`` given, beta is set so that the
    folded bias is that value."""
    out = {k: v.clone() for k, v in sd.items()}
    bn = 'I2P.backbone.' + conv_plan()[conv_index].bn_key
    out[bn + '.weight'][channel] *= torch.tensor(factor, dtype=torch.float32)
    out[bn + '.bias'][channel] *= torch.tensor(factor, dtype=torch.float32)
    if bias is not None:
        assert factor == 0, 'a chosen bias is for a zero channel'
        out[bn + '.bias'][channel] = bias              # folded bias = beta - mean * 0
    return out


def channel_max(sd: Dict[str, torch.Tensor], conv_index: int, channel: int) -> float:
    """max |folded weight| of one output channel of a conv, in float64."""
    spec = conv_plan()[conv_index]
    pre = 'I2P.backbone.'
    w = sd[pre + spec.conv_key + '.weight'][channel].double() * _bn_scale(sd, pre + spec.bn_key)[channel]
    return float(w.abs().max())


def _pow2_factors(n: int, g: torch.Generator, lo: int, hi: int) -> torch.Tensor:
    """n factors 2^k, k an integer drawn from [lo, hi], with one channel at each end of the range."""
    k = torch.randint(lo, hi + 1, (n,), generator=g)
    ends = torch.randperm(n, generator=g)[:2]
    k[ends[0]], k[ends[1]] = lo, hi
    return torch.pow(2.0, k.double()).float()


def _rescale_hidden(out, bn: str, consumers, f: torch.Tensor) -> None:
    """Multiply the BatchNorm ``bn`` (gamma and beta) by f per channel and divide input columns [c0, c0 + len(f)) of
    every consumer weight by f.  The BN is followed by a ReLU, and ReLU(f x) = f ReLU(x) for f > 0."""
    out[bn + '.weight'] *= f
    out[bn + '.bias'] *= f
    for key, c0 in consumers:
        shape = [1, -1] + [1] * (out[key].dim() - 2)
        out[key][:, c0:c0 + len(f)] /= f.view(shape)


@torch.no_grad()
def reparametrize_resnet(sd: Dict[str, torch.Tensor], seed: int, lo: int, hi: int, prefix: str = '') -> Dict[str, torch.Tensor]:
    """ResNet-50 with a wide spread of hidden-channel magnitudes: in every bottleneck, bn1's channels are scaled by
    powers of two 2^k, k in [lo, hi], and conv2's input columns divided by the same factors; likewise bn2 -> conv3.
    Powers of two make this exact in fp32: the hidden activations become exactly f * the original, and every block
    output is unchanged."""
    out = {k: v.clone() for k, v in sd.items()}
    g = torch.Generator().manual_seed(seed)
    for li, blocks in enumerate((3, 4, 6, 3), 1):
        for j in range(blocks):
            p = f'{prefix}layer{li}.{j}'
            for a, b in ((1, 2), (2, 3)):
                f = _pow2_factors(out[f'{p}.bn{a}.weight'].numel(), g, lo, hi)
                _rescale_hidden(out, f'{p}.bn{a}', [(f'{p}.conv{b}.weight', 0)], f)
    return out


@torch.no_grad()
def reparametrize_pointnet(sd: Dict[str, torch.Tensor], seed: int, lo: int, hi: int) -> Dict[str, torch.Tensor]:
    """The PointNet heads with a wide spread of hidden-channel magnitudes: each bn_i's channels scaled by powers of two
    2^k, k in [lo, hi], and the input columns of every conv that reads them divided by the same factors -- conv_{i+1};
    for bn2 also conv6's point-feature columns [0, 64); for bn5 the pooled global features, i.e. conv6's columns
    [64, 1088) (MLP_for) and all three conv6_x heads (MLP_rev).  Exact in fp32 like ``reparametrize_streams``."""
    out = {k: v.clone() for k, v in sd.items()}
    g = torch.Generator().manual_seed(seed)
    for pre, last in (('forwardDirection.', 8), ('reverseDirection.', 5)):
        for i in range(1, last + 1):
            if pre == 'forwardDirection.' and i == 5:
                consumers = [(f'{pre}conv6.weight', 64)]
            elif i == 5:
                consumers = [(f'{pre}conv6_{k}.weight', 0) for k in (1, 2, 3)]
            else:
                consumers = [(f'{pre}conv{i + 1}.weight', 0)]
                if pre == 'forwardDirection.' and i == 2:
                    consumers.append((f'{pre}conv6.weight', 0))
            f = _pow2_factors(out[f'{pre}bn{i}.weight'].numel(), g, lo, hi)
            _rescale_hidden(out, f'{pre}bn{i}', consumers, f)
    return out


def reparametrize_3dmm(pack: dict, seed: int, lo: int, hi: int) -> dict:
    """The same morphable model with a wide spread of coefficient scales: basis column k (shape and expression) is
    multiplied by 2^e_k and the whitening mean / std of coefficient k divided by it, e_k an integer in [lo, hi] (one
    coefficient at each end).  Every product W_ck alpha_k is unchanged, so the fp32 reference is bit-identical, while the
    library's alpha scales and basis row scales move."""
    import numpy as np
    rng = np.random.default_rng(seed)
    e = rng.integers(lo, hi + 1, 50)
    ends = rng.permutation(50)[:2]
    e[ends[0]], e[ends[1]] = lo, hi
    f = np.exp2(e).astype(np.float32)
    out = dict(pack)
    out['w_shp'] = pack['w_shp'] * f[:40]
    out['w_exp'] = pack['w_exp'] * f[40:]
    for key in ('param_mean', 'param_std'):
        out[key] = pack[key].copy()
        out[key][12:62] /= f
    return out


STRESS_ZERO_COEF = 45            # the coefficient of stress_3dmm with mean = std = 0


def stress_3dmm(pack: dict, seed: int = 0) -> dict:
    """A morphable model (make_3dmm format) with the rows the basis packing treats specially, in both the dense and
    the keypoint (sparse) rows: rows with u = 0, all-zero basis rows (row scale 1), rows where one column is 2^20 times
    the others, and one coefficient (``STRESS_ZERO_COEF``) with mean = std = 0, whose alpha scale is then 2^10."""
    import numpy as np
    rng = np.random.default_rng(seed)
    kp = pack['keypoints']
    n3 = pack['w_shp'].shape[0]
    pick = lambda n: np.concatenate([rng.choice(kp, n, replace=False), rng.choice(n3, 4 * n, replace=False)])
    u_shp, u_exp = pack['u_shp'].copy(), pack['u_exp'].copy()
    w = np.concatenate([pack['w_shp'], pack['w_exp']], 1)
    zero_u, zero_w, spike = pick(12), pick(12), pick(12)
    u_shp[zero_u], u_exp[zero_u] = 0.0, 0.0
    w[zero_w] = 0.0
    cols = rng.integers(0, 50, len(spike))
    w[spike, cols] *= np.float32(2.0 ** 20)
    out = dict(pack, u_shp=u_shp, u_exp=u_exp, w_shp=np.ascontiguousarray(w[:, :40]),
               w_exp=np.ascontiguousarray(w[:, 40:]))
    for key in ('param_mean', 'param_std'):
        out[key] = pack[key].copy()
        out[key][12 + STRESS_ZERO_COEF] = 0.0
    return out


def basis_arrays(n: int, seed: int):
    """(u (3n, 1), w_shp (3n, 40), w_exp (3n, 10)) fp32 with the statistics of synthetic.make_3dmm, for bases of any
    size (make_3dmm needs at least 68 vertices)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    u = (d * np.array([7.0e4, 9.0e4, 6.0e4])).reshape(-1, 1) + rng.standard_normal((3 * n, 1)) * 2.0e2
    return (u.astype(np.float32), rng.standard_normal((3 * n, 40)).astype(np.float32),
            rng.standard_normal((3 * n, 10)).astype(np.float32))


def recon_pack(base: dict, dense=None, sparse=None) -> dict:
    """Reconstruction pack (reference_port.gather_sparse_basis format) of the make_3dmm-format ``base``, with the dense
    and / or sparse basis replaced by (u, w_shp, w_exp) arrays."""
    from oracle import reference_port as rp
    out = rp.gather_sparse_basis(base)
    if dense is not None:
        out['u'], out['w_shp'], out['w_exp'] = dense
    if sparse is not None:
        out['u_base'], out['w_shp_base'], out['w_exp_base'] = sparse
    return out


@torch.no_grad()
def _calibrate_pointnet(sd: Dict[str, torch.Tensor], pooled: torch.Tensor, seed: int) -> None:
    """Same treatment for the BatchNorm1d layers of forwardDirection / reverseDirection (reference
    backbone_nets/pointnet_backbone.py:7-106): with arbitrary statistics every ReLU of the heads is dead (the
    landmark coordinates are ~100 px, the random convs scale them further) and the refinement would be identically
    zero.  Each BN gets the float64 batch statistics of its own input on a calibration batch of landmarks, perturbed,
    so that about half of the units are active at every layer."""
    import numpy as np
    from oracle import reference_port as rp
    g = torch.Generator().manual_seed(7000 + seed)
    basis = rp.gather_sparse_basis(synthetic.make_3dmm(0))
    heads = [F.linear(pooled, sd[f'I2P.backbone.{h}.1.weight'], sd[f'I2P.backbone.{h}.1.bias'])
             for h in ('classifier_ori', 'classifier_shape', 'classifier_exp')]
    attr = torch.cat(heads, 1)
    lmk = torch.from_numpy(rp.reconstruct_vertex_62(attr.numpy(), basis)).double()       # (8,3,68)

    def layer(pre, x, conv, bn):
        y = F.conv1d(x, sd[f'{pre}{conv}.weight'].double(), sd[f'{pre}{conv}.bias'].double())
        n = y.shape[1]
        mean, var = y.mean(dim=(0, 2)), y.var(dim=(0, 2), unbiased=False)
        mean = mean + 0.1 * var.sqrt() * torch.randn(n, generator=g, dtype=torch.float64)
        var = var * (0.8 + 0.4 * torch.rand(n, generator=g, dtype=torch.float64)) + 1e-6
        sd[f'{pre}{bn}.running_mean'].copy_(mean.float())
        sd[f'{pre}{bn}.running_var'].copy_(var.float())
        rm, rv = sd[f'{pre}{bn}.running_mean'].double(), sd[f'{pre}{bn}.running_var'].double()
        gamma, beta = sd[f'{pre}{bn}.weight'].double(), sd[f'{pre}{bn}.bias'].double()
        y = (y - rm.view(1, -1, 1)) / torch.sqrt(rv.view(1, -1, 1) + 1e-5) * gamma.view(1, -1, 1) + beta.view(1, -1, 1)
        return y.clamp(min=0)

    for pre in ('forwardDirection.', 'reverseDirection.'):
        out = lmk
        for i in range(1, 6):
            out = layer(pre, out, f'conv{i}', f'bn{i}')
            if i == 2:
                pf = out
        glob = out.max(dim=2, keepdim=True).values
        if pre == 'forwardDirection.':
            rep = lambda t: t.repeat(1, 1, 68)
            pool = torch.randn(lmk.shape[0], 1280, 1, generator=g, dtype=torch.float64).abs() * 0.5
            cat = torch.cat([pf, rep(glob), rep(pool), rep(attr[:, 12:52].double().unsqueeze(2)),
                             rep(attr[:, 52:62].double().unsqueeze(2))], 1)
            out = layer(pre, cat, 'conv6', 'bn6')
            for i in (7, 8, 9):
                out = layer(pre, out, f'conv{i}', f'bn{i}')
        else:
            for i in (1, 2, 3):
                layer(pre, glob, f'conv6_{i}', f'bn6_{i}')


@torch.no_grad()
def build_resnet50_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded state dict of ``resnet_backbone.resnet50()`` (reference backbone_nets/resnet_backbone.py:148-249 key
    schema, keys without prefix): kaiming convs like the reference's own init, randomised BatchNorm affine parameters
    and running statistics so that BN folding is exercised.  ReLU networks with residual connections keep their signal
    without calibration; magnitudes grow to a few hundred, which is exactly what the dynamic row scaling of the GEMM
    layers is for."""
    key = ('resnet50', seed)
    if key in _CACHE:
        return _CACHE[key]
    from synergynet_b200 import backbone
    m = backbone.resnet50()
    synthetic.seeded_init_(m, 300 + seed)
    synthetic.randomize_batchnorm_(m, 300 + seed)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    _CACHE[key] = sd
    return sd
