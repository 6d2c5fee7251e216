"""UV texture measurement: ``uv_overlay_images`` and ``uv_obj_images`` against the per-image loop of
uv_texture_realFaces.py restated on this package, in one command.
    python scripts/bench_uv.py [--counts 1,4,16] > uv_bench.json

Images: seeded synthetic.make_scene_u8 256 x 256 crops with the ROI [0, 0, 256, 256, 1.0] used as given (the script's
pre-cropped faces), one seeded 256 x 256 UV map per image, the seeded synthetic UV layout; backbone: bench.py's seeded
mobilenet_v2, INTER_LINEAR resize.  The loop arm per image: ``get_all_outputs`` with the box whose square_roi is that ROI,
the host UV gather ``np.flip(map, 0)[coord_u, coord_v][keep]``, ``Sim3DR.render(img, [m[:, keep]], deletedTri - 1,
tex=colors / 255)`` and the ``write_obj_with_colors`` format loop in memory.  The batched arm: ``uv_overlay_images`` and
``uv_obj_images`` on the whole list.  For every N, every shape is warmed up first and the arms alternate round by round,
host clock from host images to host results:
  ms_per_image   batched (overlay + OBJ) / N  x  loop / N
Medians over the rounds; `spread` is (max - min) / median.  Also printed: the card's name and power limit, and the byte
equality of the two arms (blended and solid images, OBJ text) at every N.  Fails without a GPU."""
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

SIDE = 256
ROI = [0, 0, SIDE, SIDE, 1.0]
RECT = [21.2, 21.2, 234.8, 234.8, 1.0]             # square_roi(RECT) == ROI: get_all_outputs crops the same box


def write_obj_with_colors_format(vertices, triangles, colors) -> bytes:
    """artistic.py:27-31's two format loops, joined in memory instead of written line by line."""
    s = ['v {:.4f} {:.4f} {:.4f} {} {} {}\n'.format(vertices[0, i], vertices[1, i], vertices[2, i], colors[i, 2], colors[i, 1],
                                                    colors[i, 0]) for i in range(vertices.shape[1])]
    s += ['f {} {} {}\n'.format(triangles[0, i], triangles[1, i], triangles[2, i]) for i in range(triangles.shape[1])]
    return ''.join(s).encode()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,4,16')
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('bench_uv.py needs a CUDA device (H100); nothing is measured without one')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    from synergynet_b200 import Sim3DR, synthetic
    from synergynet_b200.inference import RENDER_CFG, UVLayout, square_roi
    assert square_roi(RECT) == ROI
    model = bench.build_model(str(dev))
    model.resize_interpolation = 'linear'
    layout = UVLayout(*synthetic.make_uv_layout(0, nver=model.u.shape[0] // 3))
    out = {'workload': f'{SIDE}x{SIDE}x3 uint8 crops, ROI {ROI} as given, one {SIDE}x{SIDE} UV map per image', 'card': card(dev),
           'counts': {}}
    for n in counts:
        images = [synthetic.make_scene_u8(SIDE, SIDE, 80 + i) for i in range(n)]
        maps = [synthetic.make_uv_map(SIDE, SIDE, seed=90 + i) for i in range(n)]

        def batched():
            blended, solid = model.uv_overlay_images(images, maps, layout, rois=[ROI])
            return blended, solid, [t for faces in model.uv_obj_images(images, maps, layout, rois=[ROI]) for t in faces]

        def looped():
            blended, solid, texts = [], [], []
            for im, uv_map in zip(images, maps):
                _, meshes, _ = model.get_all_outputs(im, rects=[RECT])
                colors = np.flip(uv_map, axis=0)[layout.coord_u, layout.coord_v, :][layout.keep, :]
                m = meshes[0][:, layout.keep]
                res, overlap = Sim3DR.render(im, [m], layout.render_tri, alpha=0.6, tex=colors.astype(np.float32) / 255.0, cfg=RENDER_CFG)
                blended.append(res)
                solid.append(overlap)
                texts.append(write_obj_with_colors_format(m, layout.deleted_tri, colors.astype(np.float32)))
            return blended, solid, texts

        b, lp = batched(), looped()                        # warm-up of every shape, and the equality of the two arms
        equal = {'blended': all(np.array_equal(x, y) for x, y in zip(b[0], lp[0])),
                 'solid': all(np.array_equal(x, y) for x, y in zip(b[1], lp[1])), 'obj_bytes': b[2] == lp[2],
                 'images': n, 'text_bytes': sum(len(t) for t in b[2])}
        del b, lp
        tb, tl = [], []
        for _ in range(5 if n <= 4 else 3):
            tb.append(wall_ms(batched) / n)
            tl.append(wall_ms(looped) / n)
        stat = lambda t: {'ms_per_image': statistics.median(t), 'spread': (max(t) - min(t)) / statistics.median(t), 'rounds': len(t)}
        res = {'equal': equal, 'uv_overlay_images_plus_uv_obj_images': stat(tb), 'per_image_loop': stat(tl),
               'ratio_loop_over_batched': statistics.median(tl) / statistics.median(tb)}
        out['counts'][str(n)] = res
        print(f'[bench_uv] N={n}: ' + json.dumps(res), file=sys.stderr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
