"""Crop + resize measurement (get_all_outputs' crop stage, synergy3DMM.py:186-188):
    python scripts/bench_crop.py [--no-cpu]  > crop_bench.json

crop_img + cv2.resize to 120 x 120 of 16 face ROIs from one 720 x 1080 scene, for ROI sides 100 / 240 (the exact halving
OpenCV's INTER_LINEAR turns into its area path) / 400, in both interpolations: on the device
(inference.crop_resize_device) and as the host loop it replaced; plus get_all_outputs end to end for 16 faces.
kernel_ms = the launch alone (CUDA events over 200 launches); call_ms = host planner + plan upload + kernel, synchronised
per call.  The card's name and power limit are part of the numbers and printed with them."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def card(dev):
    """Name and power limit of the card (a read-only nvidia-smi query)."""
    try:
        q = subprocess.run(['nvidia-smi', '-i', str(dev.index), '--query-gpu=power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        q = ''
    return {'name': torch.cuda.get_device_name(dev), 'power_limit': q or 'not measured'}


def crop_measurement(dev, cpu_too=True):
    from synergynet_b200 import _lib, synthetic
    from synergynet_b200.inference import INTER_LANCZOS4, INTER_LINEAR, crop_img, crop_resize_device, resize_plan, roi_ints, square_roi
    H, W, B = 720, 1080, 16
    scene = synthetic.make_scene_u8(H, W, 0)
    img = torch.from_numpy(scene).to(dev)
    lib = _lib.load()
    out = {'workload': f'{B} ROIs of one {H}x{W}x3 uint8 scene -> planar uint8 (16,3,120,120); ROI corners on a 4 x 4 grid, '
                       'the 400 px ones reach past the image edge',
           'card': card(dev), 'cases': {}}
    for side in (100, 240, 400):
        boxes = [[40 + (i % 4) * 250, 20 + (i // 4) * 150, 40 + (i % 4) * 250 + side, 20 + (i // 4) * 150 + side] for i in range(B)]
        for name, mode in (('linear', INTER_LINEAR), ('lanczos4', INTER_LANCZOS4)):
            plan = torch.from_numpy(resize_plan(np.array([roi_ints(b) for b in boxes], np.int32), 120, 120, mode)).to(dev)
            o = torch.empty((B, 3, 120, 120), dtype=torch.uint8, device=dev)
            st = torch.cuda.current_stream(dev).cuda_stream
            launch = lambda: lib.syn_crop_resize(img.data_ptr(), H, W, 3, plan.data_ptr(), B, 120, 120, mode, o.data_ptr(),
                                                 3 * 14400, 120, 1, 14400, st)
            k_ms = bench._time_cuda(launch, iters=200, warmup=10)

            def call():
                crop_resize_device(img, boxes, (120, 120), mode)
                torch.cuda.synchronize()
            for _ in range(5):
                call()
            t0 = time.perf_counter()
            for _ in range(50):
                call()
            case = {'kernel_ms': k_ms, 'call_ms': (time.perf_counter() - t0) / 50 * 1e3}
            if cpu_too:
                import cv2
                t0, reps = time.perf_counter(), 0
                while time.perf_counter() - t0 < 1.0:
                    [cv2.resize(crop_img(scene, b), dsize=(120, 120), interpolation=mode) for b in boxes]
                    reps += 1
                case['host_loop_ms'] = (time.perf_counter() - t0) / reps * 1e3
                case['host_threads'] = cv2.getNumThreads()
            out['cases'][f'side{side}_{name}'] = case
    model = bench.build_model(str(dev))
    rng = np.random.default_rng(3)
    xy = rng.uniform([0, 0], [W - 300, H - 300], (B, 2))
    rects = [[float(x), float(y), float(x + 150), float(y + 180), 0.9] for x, y in xy]
    model.get_all_outputs(scene, rects=rects)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(20):
        model.get_all_outputs(scene, rects=rects)
    x0, _, x1, _ = roi_ints(square_roi(rects[0]))
    out['get_all_outputs'] = {'ms': (time.perf_counter() - t0) / 20 * 1e3, 'faces': B, 'interpolation': model.resize_interpolation,
                              'roi_side': x1 - x0,
                              'what': 'wall time of one call from a host uint8 image to landmarks, dense meshes and poses on the '
                                      'host (image H2D, crop + resize, backbone, reconstruction, pose, D2H)'}
    return out


if __name__ == '__main__':
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    print(json.dumps(crop_measurement(dev, cpu_too='--no-cpu' not in sys.argv)))
