"""Overlay measurement: ``overlay_batch`` against the loop a video user writes today (``get_all_outputs`` + ``Sim3DR.render``
per frame), in one command.
    python scripts/bench_overlay.py [--counts 1,4,16,64] > overlay_bench.json

Frames: seeded synthetic.make_scene_u8 scenes at 720 x 1080 (16 distinct scenes, frame i = scene i mod 16), 16 seeded rects
per frame; backbone: bench.py's seeded mobilenet_v2; triangles: synthetic.make_render_topology() (the grid topology of
the dense mesh, passed as ``connectivity`` to both arms; the synthetic parameter pack's random triangles span the whole
face and are not a mesh).  For every frame count N, every shape warmed up first and the two arms alternating round by
round, host clock from host frames to host (blended, solid) images:
  overlay_ms_per_frame   overlay_batch(frames, rects) / N x (get_all_outputs + Sim3DR.render)
Medians over the rounds; `spread` is (max - min) / median of the rounds.  Also printed: the card's name and power limit,
the bit equality of the two arms at every N, the key workspace of the frame-axis rasteriser against B x H x W x 8 bytes,
and at N = 16 (or the largest N below it) the CUDA time of each new kernel from torch.profiler in a separate run.  Fails
without a GPU."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
import bench  # noqa: E402
from bench_crop import card  # noqa: E402

H, W, FACES = 720, 1080, 16
KERNELS = ('mesh_box_kernel', 'mesh_box_scan_kernel', 'raster_depth_kernel', 'raster_resolve_frames_kernel', 'add_weighted_u8_kernel')


def wall_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def kernel_ms(fn):
    """CUDA time per launch of each new kernel in one call of fn (torch.profiler, a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
                out[k] = {'ms_total': t / 1e3, 'launches': e.count}
    return {k: out.get(k, 'not measured') for k in KERNELS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,4,16,64')
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('bench_overlay.py needs a CUDA device (H100); nothing is measured without one')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    from synergynet_b200 import Sim3DR, synthetic
    from synergynet_b200.inference import RENDER_CFG
    scenes = [synthetic.make_scene_u8(H, W, s) for s in range(16)]
    model = bench.build_model(str(dev))
    tri = synthetic.make_render_topology()
    conn = tri.T
    rng = np.random.default_rng(3)
    out = {'workload': f'{H}x{W}x3 uint8 frames, {FACES} seeded rects per frame, grid topology of {tri.shape[0]} triangles',
           'card': card(dev), 'counts': {}}
    profiled = max([n for n in counts if n <= 16] or counts[:1])
    for n in counts:
        frames = np.stack([scenes[i % 16] for i in range(n)])
        rects = [[[float(x), float(y), float(x + 150), float(y + 180), 0.9] for x, y in rng.uniform([0, 0], [W - 300, H - 300], (FACES, 2))]
                 for _ in range(n)]

        def batched():
            return model.overlay_batch(frames, rects=rects, alpha=0.6, connectivity=conn)

        def looped():
            res = []
            for i in range(n):
                _, meshes, _ = model.get_all_outputs(frames[i], rects=rects[i])
                res.append(Sim3DR.render(frames[i], meshes, tri, alpha=0.6, cfg=RENDER_CFG))
            return res
        (bb, bs), lp = batched(), looped()                 # warm-up of every shape, and the equality of the two arms
        equal = {'blended_bits': all(np.array_equal(bb[i], lp[i][0]) for i in range(n)),
                 'solid_bits': all(np.array_equal(bs[i], lp[i][1]) for i in range(n)),
                 'pixels_drawn': int((bs != frames).any(-1).sum())}
        del bb, bs, lp
        r = Sim3DR._renderer_for(np.ascontiguousarray(tri, dtype=np.int32), synthetic.NVER)
        keys = r.last_key_count
        tb, tl = [], []
        for _ in range(5 if n <= 16 else 3):
            tb.append(wall_ms(batched) / n)
            tl.append(wall_ms(looped) / n)
        stat = lambda t: {'ms_per_frame': statistics.median(t), 'spread': (max(t) - min(t)) / statistics.median(t), 'rounds': len(t)}
        res = {'equal': equal,
               'key_workspace': {'bytes': keys * 8, 'full_canvas_bytes': n * FACES * H * W * 8,
                                 'fraction': keys / float(n * FACES * H * W)},
               'overlay': {'overlay_batch': stat(tb), 'get_all_outputs_plus_render_loop': stat(tl),
                           'ratio_loop_over_batched': statistics.median(tl) / statistics.median(tb)}}
        if n == profiled:
            res['kernels_per_call'] = kernel_ms(batched)
        out['counts'][str(n)] = res
        print(f'[bench_overlay] N={n}: ' + json.dumps(res), file=sys.stderr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
