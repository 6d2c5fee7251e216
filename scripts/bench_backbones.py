#!/usr/bin/env python
"""Throughput of the conv+BN backbones on the GPU, per arch, against the same network restated in torch.nn and run
through cuDNN (fp32 with TF32 off, and with TF32 on), alternated in one process.

    python scripts/bench_backbones.py --family mbv1 [--batch 1024] [--steps 100] [--warmup 10] [--reps 3] [--archs a,b] [--out FILE]
    python scripts/bench_backbones.py --family resnet [--batch 512] [--steps 10] [--warmup 3] [--reps 2] [--archs a,b] [--out FILE]
    python scripts/bench_backbones.py --family ghostnet [--batch 1024] [--steps 50] [--warmup 10] [--reps 3] [--out FILE]

Inputs stay on the device (B normalised crops; B = 512 is the batch of BASELINE.json configs[4]); each arm is timed
with CUDA events over `steps` back-to-back forwards after `warmup` untimed ones, the arms alternate `reps` times and the
best repetition is reported.  A separate set of timed calls (syn_set_timing) gives the time per kernel kind.  Operations
are computed from the layer table here (2 x multiply-adds for TFLOP/s), and for the MobileNetV1 depthwise kernel the
bytes it must move (input map, output map, its row maxima, weights and bias); for GhostNet those of its depthwise
passes (plain and ghost mode) and of the SE gate.  Prints one JSON line per arch, with the
card's name and power limit read in the same run.  The defaults per family are those of the figures in README.md.
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ghost64, mbv1_64, resnets64, synth_ghost, synth_mbv1, synth_resnet  # noqa: E402
from oracle.gemm64 import HEADS  # noqa: E402
from synergynet_b200 import backbone, model_building, synthetic  # noqa: E402
from synergynet_b200.params import ParamsPack, set_param_pack  # noqa: E402


def conv_bn(cin, cout, k, s, sd, ck, bk, groups=1):
    conv = nn.Conv2d(cin, cout, k, s, k // 2, groups=groups, bias=False)
    bn = nn.BatchNorm2d(cout)
    conv.weight.data.copy_(sd[ck + '.weight'])
    for n in ('weight', 'bias', 'running_mean', 'running_var'):
        getattr(bn, n).data.copy_(sd[f'{bk}.{n}'])
    return conv, bn


def heads(sd, feat):
    fc = nn.Linear(feat, 102)
    fc.weight.data.copy_(torch.cat([sd[f'{h}.weight'] for h in HEADS]))
    fc.bias.data.copy_(torch.cat([sd[f'{h}.bias'] for h in HEADS]))
    return fc


# ---- MobileNetV1 ----------------------------------------------------------------------------------------------------
def mbv1_restatement(sd, arch):
    """The reference network as torch.nn modules (conv + eval BatchNorm + ReLU, avgpool, four heads) on the GPU."""
    layers = []
    for (cin, cout, k, s, g, _, _), (ck, bk) in zip(mbv1_64.stage_table(arch), backbone.mobilenet_v1_conv_keys()):
        layers += [*conv_bn(cin, cout, k, s, sd, ck, bk, g), nn.ReLU(inplace=True)]
    feat = nn.Sequential(*layers, nn.AdaptiveAvgPool2d(1), nn.Flatten())
    return nn.Sequential(feat, heads(sd, mbv1_64.stage_table(arch)[-1][1]))


def mbv1_counts(arch, batch, kinds, ms):
    """MACs by kind, and the bandwidth of the depthwise kernel: per face the bytes it must move, plus its weights."""
    t = mbv1_64.stage_table(arch)
    mac = {'stem': 0, 'dw': 0, 'pw': 0, 'heads': t[-1][1] * 102}
    dw_bytes = 0
    for i, (cin, cout, k, s, g, hi, ho) in enumerate(t):
        kind = 'stem' if i == 0 else 'dw' if i % 2 == 1 else 'pw'
        mac[kind] += ho * ho * cout * (cin // g) * k * k
        if kind == 'dw':
            dw_bytes += 4 * (hi * hi * cin + ho * ho * cout + ho * ho)
    dw_weight_bytes = sum(4 * 10 * row[1] for i, row in enumerate(t) if i % 2 == 1)
    total = sum(mac.values())
    return {
        'mmac_per_face': round(total / 1e6, 3),
        'pointwise_share_of_macs': round(mac['pw'] / total, 4),
        'algorithmic_tflops': round(2 * total * batch / ms / 1e9, 3),
        'kernel_ms': {k: round(v, 4) for k, v in kinds.items()},
        'dw_hbm_gb_per_s': round((dw_bytes * batch + dw_weight_bytes) / kinds.get('mbv1_dw3x3', float('nan')) / 1e6, 1),
    }


# ---- ResNets --------------------------------------------------------------------------------------------------------
class _RestatedResNet(nn.Module):
    """The reference network as torch.nn modules (conv + eval BatchNorm, ReLU, the shortcut adds, the pools, the four
    heads as one Linear) on the GPU."""

    def __init__(self, sd, arch):
        super().__init__()
        self.arch = arch
        self.convs = nn.ModuleList(nn.Sequential(*conv_bn(cin, cout, k, s, sd, ck, bk))
                                   for (cin, cout, k, s, _, _, _), (ck, bk)
                                   in zip(resnets64.stage_table(arch), resnets64.conv_keys(arch)))
        self.fc = heads(sd, resnets64.stage_table(arch)[-1][1])

    def forward(self, x):
        c = self.convs
        x = nn.functional.max_pool2d(torch.relu(c[0](x)), 3, 2, 1)
        for inner, last, ds in resnets64.blocks(self.arch):
            out = x
            for i in inner:
                out = torch.relu(c[i](out))
            x = torch.relu(c[last](out) + (c[ds](x) if ds is not None else x))
        return self.fc(torch.flatten(nn.functional.adaptive_avg_pool2d(x, 1), 1))


def resnet_counts(arch, batch, kinds, ms):
    """MACs of the stem, of the GEMM convs and of the heads."""
    t = resnets64.stage_table(arch)
    conv = [cin * cout * k * k * ho * ho for cin, cout, k, _, _, ho, _ in t]
    total = sum(conv) + t[-1][1] * 102
    return {
        'gmac_per_face': round(total / 1e9, 3),
        'algorithmic_tflops': round(2 * total * batch / ms / 1e9, 2),
        'kernel_ms': {k: round(v, 3) for k, v in kinds.items()},
    }


# ---- GhostNet -------------------------------------------------------------------------------------------------------
class _RestatedGhostNet(nn.Module):
    """The reference network as torch.nn modules (ghost modules, conv_dw, SE with the hard-sigmoid gate, shortcuts,
    ConvBnAct, pool, conv_head, the four heads as one Linear) on the GPU."""

    def __init__(self, sd, arch='ghostnet'):
        super().__init__()
        self.c = nn.ModuleDict()
        for ck, bk in backbone.ghostnet_conv_keys():
            w = sd[ck + '.weight']
            groups = w.shape[0] if w.shape[1] == 1 and w.shape[-1] > 1 else 1
            conv = nn.Conv2d(w.shape[1] * groups, w.shape[0], w.shape[-1], 1, w.shape[-1] // 2, groups=groups, bias=bk is None)
            conv.weight.data.copy_(w)
            mods = [conv]
            if bk is None:
                conv.bias.data.copy_(sd[ck + '.bias'])
            else:
                bn = nn.BatchNorm2d(w.shape[0])
                for n in ('weight', 'bias', 'running_mean', 'running_var'):
                    getattr(bn, n).data.copy_(sd[f'{bk}.{n}'])
                mods.append(bn)
            self.c[ck.replace('.', '_')] = nn.Sequential(*mods)
        self.fc = nn.Linear(1280, 102)
        self.fc.weight.data.copy_(torch.cat([sd[f'{h}.weight'] for h in ghost64.HEADS]))
        self.fc.bias.data.copy_(torch.cat([sd[f'{h}.bias'] for h in ghost64.HEADS]))

    def conv(self, key, x, stride=1):
        seq = self.c[key.replace('.', '_')]
        seq[0].stride = (stride, stride)
        return seq(x)

    def ghost(self, key, x, relu):
        x1 = self.conv(key + '.primary_conv.0', x)
        x1 = torch.relu(x1) if relu else x1
        x2 = self.conv(key + '.cheap_operation.0', x1)
        return torch.cat([x1, torch.relu(x2) if relu else x2], dim=1)

    def forward(self, x):
        x = torch.relu(self.conv('conv_stem', x, 2))
        for b in ghost64.blocks():
            p = b['p']
            y = self.ghost(p + 'ghost1', x, True)
            if b['s'] > 1:
                y = self.conv(p + 'conv_dw', y, b['s'])
            if b['red']:
                z = self.conv(p + 'se.conv_expand', torch.relu(self.conv(p + 'se.conv_reduce', y.mean((2, 3), keepdim=True))))
                y = y * nn.functional.relu6(z + 3.0) / 6.0
            y = self.ghost(p + 'ghost2', y, False)
            x = y + (self.conv(p + 'shortcut.2', self.conv(p + 'shortcut.0', x, b['s'])) if b['short'] else x)
        x = torch.relu(self.conv('blocks.9.0.conv', x)).mean((2, 3), keepdim=True)
        return self.fc(torch.flatten(torch.relu(self.conv('conv_head', x)), 1))


def ghost_counts(arch, batch, kinds, ms):
    """MACs by kind, and the bandwidth of the depthwise passes and of the SE gate: per face the bytes each must move."""
    mac = {'stem': 27 * 16 * 3600, 'pw': 0, 'dw': 0, 'heads': 1280 * 102}
    dw_bytes = se_bytes = 0
    for b in ghost64.blocks():
        P, PO, i1, i2 = b['h'] ** 2, b['ho'] ** 2, b['mid'] // 2, b['cout'] // 2
        mac['pw'] += P * b['cin'] * i1 + PO * b['mid'] * i2 + 2 * b['mid'] * b['red']
        mac['dw'] += 9 * (P * i1 + PO * i2)
        dw_bytes += 4 * (P * i1 + P * b['mid'] + P + PO * i2 + PO * b['cout'] + PO + PO * b['cout'])   # ghost passes
        if b['s'] > 1:
            mac['dw'] += b['k'] ** 2 * PO * b['mid']
            dw_bytes += 4 * (P * b['mid'] + PO * b['mid'] + PO)
        if b['short']:
            mac['pw'] += PO * b['cin'] * b['cout']
            mac['dw'] += b['k'] ** 2 * PO * b['cin']
            dw_bytes += 4 * (P * b['cin'] + PO * b['cin'] + PO)
        if b['red']:
            se_bytes += 4 * (2 * PO * b['mid'] + PO + b['mid'])
    mac['pw'] += 16 * 160 * 960 + 960 * 1280
    total = sum(mac.values())
    dw_ms = sum(kinds.get(k, 0.0) for k in ('ghost_cheap', 'ghost_cheap_add', 'ghost_dw', 'ghost_shortcut_dw'))
    return {
        'mmac_per_face': round(total / 1e6, 3),
        'algorithmic_tflops': round(2 * total * batch / ms / 1e9, 3),
        'kernel_ms': {k: round(v, 4) for k, v in kinds.items()},
        'dw_hbm_gb_per_s': round(dw_bytes * batch / dw_ms / 1e6, 1) if dw_ms else None,
        'se_apply_hbm_gb_per_s': round(se_bytes * batch / kinds['ghost_se_apply'] / 1e6, 1) if 'ghost_se_apply' in kinds else None,
    }


def ghost_engine(sd, arch, dev):
    m = backbone.ghostnet()
    m.load_state_dict(sd, strict=True)
    return m.eval()._engine(dev), m


# per family: archs, defaults, checkpoint, restatement, forward, timed calls, kernel-kind name, counts, digits of ms
FAMILIES = {
    'mbv1': dict(archs=backbone.MBV1_WIDTHS, batch=1024, steps=100, warmup=10, reps=3,
                 checkpoint=synth_mbv1.build_mobilenet_v1_state_dict, restate=mbv1_restatement,
                 forward=lambda eng, x: eng.forward_mobilenet_v1(x), timed_calls=20,
                 kind=lambda n: 'mbv1_conv_sep' if n.startswith('mbv1_conv_sep') else n, counts=mbv1_counts, digits=4),
    'resnet': dict(archs=backbone.RESNET_ARCHS, batch=512, steps=10, warmup=3, reps=2,
                   checkpoint=synth_resnet.build_resnet_state_dict, restate=_RestatedResNet,
                   forward=lambda eng, x: eng.forward_resnet(x), timed_calls=5,
                   kind=lambda n: n, counts=resnet_counts, digits=3),
    'ghostnet': dict(archs={'ghostnet': None}, batch=1024, steps=50, warmup=10, reps=3,
                     checkpoint=lambda seed, arch: synth_ghost.build_ghostnet_state_dict(seed), restate=_RestatedGhostNet,
                     forward=lambda eng, x: eng.forward_ghostnet(x), timed_calls=20,
                     kind=lambda n: n, counts=ghost_counts, digits=4, engine=ghost_engine),
}


def time_arm(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:       # the number is still reported, with what is known about the card
        q = f'unavailable ({e})'
    return name, q


def set_tf32(on):
    torch.backends.cudnn.allow_tf32 = on
    torch.backends.cuda.matmul.allow_tf32 = on


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--family', choices=sorted(FAMILIES), required=True)
    ap.add_argument('--batch', type=int)
    ap.add_argument('--steps', type=int)
    ap.add_argument('--warmup', type=int)
    ap.add_argument('--reps', type=int)
    ap.add_argument('--archs')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    fam = FAMILIES[a.family]
    for k in ('batch', 'steps', 'warmup', 'reps'):
        if getattr(a, k) is None:
            setattr(a, k, fam[k])
    archs = a.archs.split(',') if a.archs else list(fam['archs'])
    if not torch.cuda.is_available():
        raise SystemExit('bench_backbones.py needs a CUDA device (H100); nothing is measured without one')
    set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))
    name, power = card()
    dev = torch.device('cuda', 0)
    x = synthetic.normalize_crops(synthetic.make_crops_u8(a.batch, seed=5)).to(dev)
    d = fam['digits']
    lines = []
    for arch in archs:
        sd = fam['checkpoint'](0, arch)
        if 'engine' in fam:
            eng, m = fam['engine'](sd, arch, dev)
        else:
            m = model_building.SynergyNet(types.SimpleNamespace(arch=arch, img_size=120, devices_id=[0]))
            m.load_state_dict({'I2P.backbone.' + k: v for k, v in sd.items()}, strict=False)
            eng = m._engine(dev)
        ref = fam['restate'](sd, arch).cuda().eval()
        ours = lambda: fam['forward'](eng, x)
        with torch.no_grad():
            got = ours()[0]
            set_tf32(False)
            want = ref(x)
            err = float((got - want).abs().max() / want.abs().max())
            best = {'ours': 1e30, 'cudnn_fp32': 1e30, 'cudnn_tf32': 1e30}
            for _ in range(a.reps):
                best['ours'] = min(best['ours'], time_arm(ours, a.steps, a.warmup))
                for tf32 in (False, True):
                    set_tf32(tf32)
                    key = 'cudnn_tf32' if tf32 else 'cudnn_fp32'
                    best[key] = min(best[key], time_arm(lambda: ref(x), a.steps, a.warmup))
            set_tf32(False)
        # time per kernel kind: mean over the timed calls
        kinds, calls = {}, fam['timed_calls']
        eng.set_timing(True)
        for _ in range(calls):
            fam['forward'](eng, x)
            for n, ms in eng.timings(max_entries=256):
                k = fam['kind'](n)
                kinds[k] = kinds.get(k, 0.0) + ms / calls
        eng.set_timing(False)
        assert eng.poll_error() == 0
        line = {
            'arch': arch, 'batch': a.batch, 'steps': a.steps, 'reps': a.reps,
            'ms_per_batch': round(best['ours'], d), 'faces_per_s': round(a.batch / best['ours'] * 1e3),
            'cudnn_fp32_ms': round(best['cudnn_fp32'], d), 'cudnn_tf32_ms': round(best['cudnn_tf32'], d),
            'speedup_vs_cudnn_fp32': round(best['cudnn_fp32'] / best['ours'], 3),
            'speedup_vs_cudnn_tf32': round(best['cudnn_tf32'] / best['ours'], 3),
            'out102_rel_err_vs_cudnn_fp32': err,
            **fam['counts'](arch, a.batch, kinds, best['ours']),
            'gpu': name, 'power_limit_max_sm_clock': power,
        }
        print(json.dumps(line), flush=True)
        lines.append(line)
        del eng, m, ref
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
