#!/usr/bin/env python
"""Throughput of the MobileNetV1 backbones on the GPU, per width, against the same network restated in torch.nn and run
through cuDNN (fp32 with TF32 off, and with TF32 on), alternated in one process.

    python scripts/bench_mbv1.py [--batch 1024] [--steps 100] [--warmup 10] [--reps 3] [--out FILE]

Inputs stay on the device (B normalised crops); each arm is timed with CUDA events over `steps` back-to-back forwards
after `warmup` untimed ones, the arms alternate `reps` times and the best repetition is reported.  A separate timed
call (syn_set_timing) gives the time per kernel kind.  Operations and bytes are computed from the layer table here:
2 x multiply-adds for TFLOP/s, and for the depthwise kernel the bytes it must move (input map, output map, its row
maxima, weights and bias).  Prints one JSON line per width, with the card's name and power limit read in the same run.
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
from oracle import mbv1_64, synth_mbv1  # noqa: E402
from synergynet_b200 import backbone, model_building, synthetic  # noqa: E402
from synergynet_b200.params import ParamsPack, set_param_pack  # noqa: E402


def layer_counts(arch):
    """Per face: multiply-adds by kind, and bytes the depthwise kernel moves."""
    t = mbv1_64.stage_table(arch)
    mac = {'stem': 0, 'dw': 0, 'pw': 0, 'heads': 0}
    dw_bytes = 0
    for i, (cin, cout, k, s, g, hi, ho) in enumerate(t):
        kind = 'stem' if i == 0 else 'dw' if i % 2 == 1 else 'pw'
        mac[kind] += ho * ho * cout * (cin // g) * k * k
        if kind == 'dw':
            dw_bytes += 4 * (hi * hi * cin + ho * ho * cout + ho * ho)
    mac['heads'] = t[-1][1] * 102
    return mac, dw_bytes


def dw_weight_bytes(arch):
    return sum(4 * 10 * row[1] for i, row in enumerate(mbv1_64.stage_table(arch)) if i % 2 == 1)


def torch_restatement(sd, arch):
    """The reference network as torch.nn modules (conv + eval BatchNorm + ReLU, avgpool, four heads) on the GPU."""
    layers = []
    for (cin, cout, k, s, g, _, _), (ck, bk) in zip(mbv1_64.stage_table(arch), backbone.mobilenet_v1_conv_keys()):
        conv = nn.Conv2d(cin, cout, k, s, k // 2, groups=g, bias=False)
        bn = nn.BatchNorm2d(cout)
        conv.weight.data.copy_(sd[ck + '.weight'])
        for n in ('weight', 'bias', 'running_mean', 'running_var'):
            getattr(bn, n).data.copy_(sd[f'{bk}.{n}'])
        layers += [conv, bn, nn.ReLU(inplace=True)]
    feat = nn.Sequential(*layers, nn.AdaptiveAvgPool2d(1), nn.Flatten())
    fc = nn.Linear(mbv1_64.stage_table(arch)[-1][1], 102)
    fc.weight.data.copy_(torch.cat([sd[f'{h}.weight'] for h in mbv1_64.HEADS]))
    fc.bias.data.copy_(torch.cat([sd[f'{h}.bias'] for h in mbv1_64.HEADS]))
    return nn.Sequential(feat, fc).cuda().eval()


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=1024)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--archs', default=','.join(backbone.MBV1_WIDTHS))
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mbv1.py needs a CUDA device (H100); nothing is measured without one')
    set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))
    name, power = card()
    dev = torch.device('cuda', 0)
    x = synthetic.normalize_crops(synthetic.make_crops_u8(a.batch, seed=5)).to(dev)
    lines = []
    for arch in a.archs.split(','):
        sd = synth_mbv1.build_mobilenet_v1_state_dict(0, arch)
        m = model_building.SynergyNet(types.SimpleNamespace(arch=arch, img_size=120, devices_id=[0]))
        m.load_state_dict({'I2P.backbone.' + k: v for k, v in sd.items()}, strict=False)
        eng = m._engine(dev)
        ref = torch_restatement(sd, arch)
        ours = lambda: eng.forward_mobilenet_v1(x)
        with torch.no_grad():
            got = ours()[0]
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cuda.matmul.allow_tf32 = False
            want = ref(x)
            err = float((got - want).abs().max() / want.abs().max())
            best = {'ours': 1e30, 'cudnn_fp32': 1e30, 'cudnn_tf32': 1e30}
            for _ in range(a.reps):
                best['ours'] = min(best['ours'], time_arm(ours, a.steps, a.warmup))
                for tf32 in (False, True):
                    torch.backends.cudnn.allow_tf32 = tf32
                    torch.backends.cuda.matmul.allow_tf32 = tf32
                    key = 'cudnn_tf32' if tf32 else 'cudnn_fp32'
                    best[key] = min(best[key], time_arm(lambda: ref(x), a.steps, a.warmup))
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cuda.matmul.allow_tf32 = False
        # time per kernel kind: mean over 20 timed calls
        kinds = {}
        eng.set_timing(True)
        for _ in range(20):
            eng.forward_mobilenet_v1(x)
            for n, ms in eng.timings():
                k = 'mbv1_conv_sep' if n.startswith('mbv1_conv_sep') else n
                kinds[k] = kinds.get(k, 0.0) + ms / 20
        eng.set_timing(False)
        mac, dw_bytes = layer_counts(arch)
        flops = 2 * sum(mac.values()) * a.batch
        dw_ms = kinds.get('mbv1_dw3x3', float('nan'))
        line = {
            'arch': arch, 'batch': a.batch, 'steps': a.steps, 'reps': a.reps,
            'ms_per_batch': round(best['ours'], 4), 'faces_per_s': round(a.batch / best['ours'] * 1e3),
            'cudnn_fp32_ms': round(best['cudnn_fp32'], 4), 'cudnn_tf32_ms': round(best['cudnn_tf32'], 4),
            'speedup_vs_cudnn_fp32': round(best['cudnn_fp32'] / best['ours'], 3),
            'speedup_vs_cudnn_tf32': round(best['cudnn_tf32'] / best['ours'], 3),
            'out102_rel_err_vs_cudnn_fp32': err,
            'mmac_per_face': round(sum(mac.values()) / 1e6, 3),
            'pointwise_share_of_macs': round(mac['pw'] / sum(mac.values()), 4),
            'algorithmic_tflops': round(flops / best['ours'] / 1e9, 3),
            'kernel_ms': {k: round(v, 4) for k, v in kinds.items()},
            'dw_hbm_gb_per_s': round((dw_bytes * a.batch + dw_weight_bytes(arch)) / dw_ms / 1e6, 1),
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
