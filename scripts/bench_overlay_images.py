"""Image-list overlay measurement: ``overlay_images`` against the loop a user with a folder of photos writes today
(``get_all_outputs`` + ``Sim3DR.render`` per image), in one command.
    python scripts/bench_overlay_images.py [--counts 1,4,16,64] > overlay_images_bench.json

Images: seeded synthetic.make_scene_u8 scenes with sizes drawn (seed 5) from bench_images.py's five sizes (450x450,
480x640, 720x1080, 1080x1920, 300x400), 16 seeded rects per image; backbone: bench.py's seeded mobilenet_v2; triangles:
synthetic.make_render_topology(), passed as ``connectivity`` to both arms.  For every image count N, every shape warmed up
first and the two arms alternating round by round, host clock from host images to host (blended, solid) images:
  overlay_ms_per_image   overlay_images(images, rects) / N x (get_all_outputs + Sim3DR.render)
Medians over the rounds; `spread` is (max - min) / median of the rounds.  Also printed: the card's name and power limit,
the bit equality of the two arms at every N, and the key workspace of the image-list rasteriser against padding every
image to the largest one (N x 16 x H_max x W_max x 8 bytes).  Fails without a GPU."""
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
from bench_frames import wall_ms  # noqa: E402
from bench_images import FACES, MIX  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,4,16,64')
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('bench_overlay_images.py needs a CUDA device (H100); nothing is measured without one')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    from synergynet_b200 import Sim3DR, synthetic
    from synergynet_b200.inference import RENDER_CFG
    model = bench.build_model(str(dev))
    tri = synthetic.make_render_topology()
    conn = tri.T
    rng = np.random.default_rng(5)
    out = {'workload': f'uint8 images of sizes drawn from {list(MIX)}, {FACES} seeded rects per image, grid topology of '
                       f'{tri.shape[0]} triangles', 'card': card(dev), 'counts': {}}
    for n in counts:
        sizes = [MIX[int(k)] for k in rng.integers(0, len(MIX), n)]
        images = [synthetic.make_scene_u8(h, w, 100 + i) for i, (h, w) in enumerate(sizes)]
        rects = [[[float(x), float(y), float(x + 150), float(y + 180), 0.9]
                  for x, y in rng.uniform([0, 0], [max(w - 300, 1), max(h - 300, 1)], (FACES, 2))] for h, w in sizes]

        def batched():
            return model.overlay_images(images, rects=rects, alpha=0.6, connectivity=conn)

        def looped():
            res = []
            for i in range(n):
                _, meshes, _ = model.get_all_outputs(images[i], rects=rects[i])
                res.append(Sim3DR.render(images[i], meshes, tri, alpha=0.6, cfg=RENDER_CFG))
            return res
        (bb, bs), lp = batched(), looped()                 # warm-up of every shape, and the equality of the two arms
        equal = {'blended_bits': all(np.array_equal(bb[i], lp[i][0]) for i in range(n)),
                 'solid_bits': all(np.array_equal(bs[i], lp[i][1]) for i in range(n)),
                 'pixels_drawn': int(sum((bs[i] != images[i]).any(-1).sum() for i in range(n)))}
        del bb, bs, lp
        r = Sim3DR._renderer_for(np.ascontiguousarray(tri, dtype=np.int32), synthetic.NVER)
        keys = r.last_key_count
        padded = n * FACES * max(h for h, w in sizes) * max(w for h, w in sizes)
        tb, tl = [], []
        for _ in range(5 if n <= 16 else 3):
            tb.append(wall_ms(batched) / n)
            tl.append(wall_ms(looped) / n)
        stat = lambda t: {'ms_per_image': statistics.median(t), 'spread': (max(t) - min(t)) / statistics.median(t), 'rounds': len(t)}
        res = {'sizes': [f'{h}x{w}' for h, w in sizes], 'equal': equal,
               'key_workspace': {'bytes': keys * 8, 'padded_to_largest_bytes': padded * 8, 'fraction': keys / float(padded)},
               'overlay': {'overlay_images': stat(tb), 'get_all_outputs_plus_render_loop': stat(tl),
                           'ratio_loop_over_batched': statistics.median(tl) / statistics.median(tb)}}
        out['counts'][str(n)] = res
        print(f'[bench_overlay_images] N={n}: ' + json.dumps({k: res[k] for k in ('equal', 'key_workspace', 'overlay')}), file=sys.stderr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
