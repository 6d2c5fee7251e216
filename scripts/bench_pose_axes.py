"""Pose-axis measurement: ``pose_overlay_batch`` against the loop a video user writes today (``get_all_outputs_batch``,
then the same end points drawn with host ``cv2.line`` frame by frame), in one command.
    python scripts/bench_pose_axes.py [--counts 1,4,16,64] > pose_axes_bench.json

Frames: seeded synthetic.make_scene_u8 scenes at 720 x 1080 (16 distinct scenes, frame i = scene i mod 16), 16 seeded rects
per frame; backbone: bench.py's seeded mobilenet_v2.  For every frame count N, every shape warmed up first and the two
arms alternating round by round, host clock from host frames to host pose images:
  pose_ms_per_frame   pose_overlay_batch(frames, rects) / N x (get_all_outputs_batch + plan_axis + cv2.line per face)
Medians over the rounds; `spread` is (max - min) / median of the rounds.  Also printed: the card's name and power limit,
the byte equality of the two arms at every N, and at N = 16 (or the largest N below it) the CUDA time of
draw_lines_kernel from torch.profiler in a separate run.  Fails without a GPU."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
import bench  # noqa: E402
from bench_crop import card  # noqa: E402
from bench_overlay import wall_ms  # noqa: E402

H, W, FACES = 720, 1080, 16
KERNEL = 'draw_lines_kernel'


def kernel_ms(fn):
    """CUDA time of draw_lines_kernel in one call of fn (torch.profiler, a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if KERNEL in e.key:
            t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
            return {'ms_total': t / 1e3, 'launches': e.count}
    return 'not measured'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,4,16,64')
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('bench_pose_axes.py needs a CUDA device (H100); nothing is measured without one')
    import cv2
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    from synergynet_b200 import synthetic
    from synergynet_b200.inference import plan_axis
    scenes = [synthetic.make_scene_u8(H, W, s) for s in range(16)]
    model = bench.build_model(str(dev))
    rng = np.random.default_rng(3)
    out = {'workload': f'{H}x{W}x3 uint8 frames, {FACES} seeded rects per frame', 'card': card(dev), 'counts': {}}
    profiled = max([n for n in counts if n <= 16] or counts[:1])
    for n in counts:
        frames = np.stack([scenes[i % 16] for i in range(n)])
        rects = [[[float(x), float(y), float(x + 150), float(y + 180), 0.9] for x, y in rng.uniform([0, 0], [W - 300, H - 300], (FACES, 2))]
                 for _ in range(n)]

        def batched():
            return model.pose_overlay_batch(frames, rects=rects)

        def looped():
            res = []
            for i, (lmks, _, poses) in enumerate(model.get_all_outputs_batch(frames, rects=rects)):
                img = frames[i].copy()
                for (angles, _), lmk in zip(poses, lmks):
                    segs, err = plan_axis(angles[0], angles[1], angles[2], lmk)
                    for x0, y0, x1, y1, colour in segs:
                        cv2.line(img, (x0, y0), (x1, y1), colour, 4)
                    if err is not None:
                        raise err
                res.append(img)
            return res
        b, lp = batched(), looped()                        # warm-up of every shape, and the equality of the two arms
        equal = {'bits': all(np.array_equal(b[i], lp[i]) for i in range(n)), 'pixels_drawn': int((b != frames).any(-1).sum())}
        del b, lp
        tb, tl = [], []
        for _ in range(7 if n <= 16 else 5):
            tb.append(wall_ms(batched) / n)
            tl.append(wall_ms(looped) / n)
        stat = lambda t: {'ms_per_frame': statistics.median(t), 'spread': (max(t) - min(t)) / statistics.median(t), 'rounds': len(t)}
        res = {'equal': equal,
               'pose': {'pose_overlay_batch': stat(tb), 'get_all_outputs_batch_plus_cv2_line_loop': stat(tl),
                        'ratio_loop_over_batched': statistics.median(tl) / statistics.median(tb)}}
        if n == profiled:
            res['draw_kernel_per_call'] = kernel_ms(batched)
        out['counts'][str(n)] = res
        print(f'[bench_pose_axes] N={n}: ' + json.dumps(res), file=sys.stderr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
