#!/usr/bin/env python
"""Throughput of the ResNet backbones on the GPU, per arch, against the same network restated in torch.nn and run through
cuDNN (fp32 with TF32 off, and with TF32 on), alternated in one process.

    python scripts/bench_resnets.py [--batch 512] [--steps 10] [--warmup 3] [--reps 2] [--archs a,b] [--out FILE]

Inputs stay on the device (B normalised crops; B = 512 is the batch of BASELINE.json configs[4]); each arm is timed with
CUDA events over `steps` back-to-back forwards after `warmup` untimed ones, the arms alternate `reps` times and the best
repetition is reported.  A separate set of timed calls (syn_set_timing) gives the time per kernel kind.  Operations are
computed from the layer table here (2 x multiply-adds for TFLOP/s).  Prints one JSON line per arch, with the card's name
and power limit read in the same run.
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
from oracle import resnets64, synth_resnet  # noqa: E402
from oracle.gemm64 import HEADS  # noqa: E402
from synergynet_b200 import backbone, model_building, synthetic  # noqa: E402
from synergynet_b200.params import ParamsPack, set_param_pack  # noqa: E402


def macs(arch):
    """Per face: multiply-adds of the stem, of the GEMM convs and of the heads."""
    t = resnets64.stage_table(arch)
    conv = [cin * cout * k * k * ho * ho for cin, cout, k, _, _, ho, _ in t]
    return {'stem': conv[0], 'convs': sum(conv[1:]), 'heads': t[-1][1] * 102}


class _Restated(nn.Module):
    """The reference network as torch.nn modules (conv + eval BatchNorm, ReLU, the shortcut adds, the pools, the four
    heads as one Linear) on the GPU."""

    def __init__(self, sd, arch):
        super().__init__()
        self.arch = arch
        self.convs = nn.ModuleList()
        for (cin, cout, k, s, _, _, _), (ck, bk) in zip(resnets64.stage_table(arch), resnets64.conv_keys(arch)):
            conv = nn.Conv2d(cin, cout, k, s, k // 2, bias=False)
            bn = nn.BatchNorm2d(cout)
            conv.weight.data.copy_(sd[ck + '.weight'])
            for n in ('weight', 'bias', 'running_mean', 'running_var'):
                getattr(bn, n).data.copy_(sd[f'{bk}.{n}'])
            self.convs.append(nn.Sequential(conv, bn))
        self.fc = nn.Linear(resnets64.stage_table(arch)[-1][1], 102)
        self.fc.weight.data.copy_(torch.cat([sd[f'{h}.weight'] for h in HEADS]))
        self.fc.bias.data.copy_(torch.cat([sd[f'{h}.bias'] for h in HEADS]))

    def forward(self, x):
        c = self.convs
        x = nn.functional.max_pool2d(torch.relu(c[0](x)), 3, 2, 1)
        for inner, last, ds in resnets64.blocks(self.arch):
            out = x
            for i in inner:
                out = torch.relu(c[i](out))
            x = torch.relu(c[last](out) + (c[ds](x) if ds is not None else x))
        return self.fc(torch.flatten(nn.functional.adaptive_avg_pool2d(x, 1), 1))


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
    ap.add_argument('--batch', type=int, default=512)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--archs', default=','.join(backbone.RESNET_ARCHS))
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_resnets.py needs a CUDA device (H100); nothing is measured without one')
    set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))
    name, power = card()
    dev = torch.device('cuda', 0)
    x = synthetic.normalize_crops(synthetic.make_crops_u8(a.batch, seed=5)).to(dev)
    lines = []
    for arch in a.archs.split(','):
        sd = synth_resnet.build_resnet_state_dict(0, arch)
        m = model_building.SynergyNet(types.SimpleNamespace(arch=arch, img_size=120, devices_id=[0]))
        m.load_state_dict({'I2P.backbone.' + k: v for k, v in sd.items()}, strict=False)
        eng = m._engine(dev)
        ref = _Restated(sd, arch).cuda().eval()
        ours = lambda: eng.forward_resnet(x)
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
        # time per kernel kind: mean over 5 timed calls
        kinds, calls = {}, 5
        eng.set_timing(True)
        for _ in range(calls):
            eng.forward_resnet(x)
            for n, ms in eng.timings(max_entries=256):
                kinds[n] = kinds.get(n, 0.0) + ms / calls
        eng.set_timing(False)
        assert eng.poll_error() == 0
        mac = macs(arch)
        flops = 2 * sum(mac.values()) * a.batch
        line = {
            'arch': arch, 'batch': a.batch, 'steps': a.steps, 'reps': a.reps,
            'ms_per_batch': round(best['ours'], 3), 'faces_per_s': round(a.batch / best['ours'] * 1e3),
            'cudnn_fp32_ms': round(best['cudnn_fp32'], 3), 'cudnn_tf32_ms': round(best['cudnn_tf32'], 3),
            'speedup_vs_cudnn_fp32': round(best['cudnn_fp32'] / best['ours'], 3),
            'speedup_vs_cudnn_tf32': round(best['cudnn_tf32'] / best['ours'], 3),
            'out102_rel_err_vs_cudnn_fp32': err,
            'gmac_per_face': round(sum(mac.values()) / 1e9, 3),
            'algorithmic_tflops': round(flops / best['ours'] / 1e9, 2),
            'kernel_ms': {k: round(v, 3) for k, v in kinds.items()},
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
