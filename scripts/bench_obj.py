"""OBJ measurement: ``obj_images`` against the loop a user writes today (``get_all_outputs_images``, then the reference's
write_obj format strings per face, in memory), in one command.
    python scripts/bench_obj.py [--counts 1,4,16] > obj_bench.json

Images: seeded synthetic.make_scene_u8 scenes at 720 x 1080, one seeded rect per face, four faces per image (fewer for
N < 4); backbone: bench.py's seeded mobilenet_v2; triangles: the model's (3, ntri) list + 1.  For every face count N,
every shape warmed up first and the two arms alternating round by round, host clock from host images to a list of
``bytes`` per face:
  ms_per_face       obj_images(images, rects) / N  x  (get_all_outputs_images + the write_obj format loop per face)
  text_MB_per_s     the output bytes over each arm's time
Medians over the rounds; `spread` is (max - min) / median of the rounds.  Also printed: the card's name and power limit,
the byte equality of the two arms at every N, and at the largest N the CUDA time of the OBJ kernels and of the
device-to-host copies from torch.profiler in a separate run.  Fails without a GPU."""
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

H, W, PER_IMAGE = 720, 1080, 4


def reference_format(vertices, triangles) -> bytes:
    """utils/inference.py:17-23's two format loops, joined in memory instead of written line by line."""
    s = ['v {:.4f} {:.4f} {:.4f}\n'.format(vertices[0, i], vertices[1, i], vertices[2, i]) for i in range(vertices.shape[1])]
    s += ['f {} {} {}\n'.format(triangles[2, i], triangles[1, i], triangles[0, i]) for i in range(triangles.shape[1])]
    return ''.join(s).encode()


def device_ms(fn):
    """CUDA time of the obj_* kernels and of the device-to-host copies in one call of fn (torch.profiler, a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = (getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)) / 1e3
        if 'obj_' in e.key and 'kernel' in e.key:
            out[e.key.split('(')[0]] = {'ms_total': t, 'launches': e.count}
        elif 'Memcpy DtoH' in e.key:
            out['memcpy_dtoh'] = {'ms_total': t, 'count': e.count}
    return out or 'not measured'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,4,16')
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('bench_obj.py needs a CUDA device (H100); nothing is measured without one')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    from synergynet_b200 import synthetic
    model = bench.build_model(str(dev))
    tri = model.triangles.cpu().numpy() + 1
    rng = np.random.default_rng(5)
    out = {'workload': f'{H}x{W}x3 uint8 images, {PER_IMAGE} seeded rects per image, write_obj format', 'card': card(dev),
           'counts': {}}
    for n in counts:
        per = [min(PER_IMAGE, n - k) for k in range(0, n, PER_IMAGE)]
        images = [synthetic.make_scene_u8(H, W, 40 + i) for i in range(len(per))]
        rects = [[[float(x), float(y), float(x + 200), float(y + 220), 0.9] for x, y in rng.uniform([0, 0], [W - 300, H - 300], (c, 2))]
                 for c in per]

        def batched():
            return [t for faces in model.obj_images(images, rects=rects) for t in faces]

        def looped():
            return [reference_format(mesh, tri) for _, meshes, _ in model.get_all_outputs_images(images, rects=rects) for mesh in meshes]
        b, lp = batched(), looped()                        # warm-up of every shape, and the equality of the two arms
        n_bytes = sum(len(t) for t in b)
        equal = {'bytes': b == lp, 'faces': len(b), 'text_bytes': n_bytes}
        del b, lp
        tb, tl = [], []
        for _ in range(5 if n <= 4 else 3):
            tb.append(wall_ms(batched) / n)
            tl.append(wall_ms(looped) / n)
        stat = lambda t: {'ms_per_face': statistics.median(t), 'spread': (max(t) - min(t)) / statistics.median(t), 'rounds': len(t),
                          'text_MB_per_s': n_bytes / n / statistics.median(t) / 1e3}
        res = {'equal': equal, 'obj': {'obj_images': stat(tb), 'get_all_outputs_images_plus_format_loop': stat(tl),
                                       'ratio_loop_over_device': statistics.median(tl) / statistics.median(tb)}}
        if n == max(counts):
            res['device_per_call'] = device_ms(batched)
        out['counts'][str(n)] = res
        print(f'[bench_obj] N={n}: ' + json.dumps(res), file=sys.stderr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
