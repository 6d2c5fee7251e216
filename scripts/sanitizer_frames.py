#!/usr/bin/env python
"""The frame-batch and image-list paths for `compute-sanitizer --tool memcheck` / `--tool racecheck` (needs an H100): one
batched detector pass on frames whose maps make 64-row tiles straddle frames, one ``detect_batch`` with the device
shrink, one ``get_all_outputs_batch`` with ROIs over the frame edges and a frame without a face; then the same on a list of
images of different sizes (1 x 1 images sharing a tile, two oversized images shrunk by different scales), and one
``overlay_images`` over a 1 x 1 image, faces across their own image's edges and a dense chunk that ends inside an image.
scripts/sanitizer_smoke.py covers the one-image kernels."""
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import synth_model  # noqa: E402
from synergynet_b200 import faceboxes, model_building, synthetic  # noqa: E402
from synergynet_b200.params import ParamsPack, set_param_pack  # noqa: E402


def main():
    set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))
    det = faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0), device='cuda:0')
    frames = np.stack([synthetic.make_scene_u8(193, 258, s) for s in range(3)])
    loc, conf = det.net.forward_batch(torch.from_numpy(frames).cuda())
    boxes = det.detect_batch(frames)
    big = det.detect_batch(np.stack([synthetic.make_scene_u8(750, 1100, s) for s in range(2)]))     # shrunk on the device
    m = model_building.SynergyNet(types.SimpleNamespace(arch='mobilenet_v2', img_size=120, devices_id=[0]))
    m.load_state_dict(synth_model.build_state_dict(0), strict=True)
    m.eval()
    rects = [[[-10.0, -5.0, 50.0, 55.0, 0.9], [150.0, 120.0, 300.0, 230.0, 0.8]], [], [[40.0, 20.0, 100.0, 80.0, 0.7]]]
    out = m.get_all_outputs_batch(frames, rects=rects)
    sizes = [(193, 258), (1, 1), (1, 333), (1, 1), (750, 1100), (1500, 900), (97, 61)]
    images = [synthetic.make_scene_u8(h, w, s) for s, (h, w) in enumerate(sizes)]
    small = [torch.from_numpy(im).cuda() for im in images if im.shape[0] <= 720 and im.shape[1] <= 1080]
    loc_i, _ = det.net.forward_images(small)
    boxes_i = det.detect_images(images)
    rects_i = [rects[0], [], rects[2], [], [[600.0, 650.0, 1200.0, 780.0, 0.9]], [], [[-3.0, -3.0, 80.0, 70.0, 0.9]]]
    out_i = m.get_all_outputs_images(images, rects=rects_i)
    # overlay_images: a 1 x 1 image with a face, faces across their own image's edges, and dense chunks of two faces, so
    # that a chunk ends inside image 0 and the next spans images 0 and 1
    ov_images = [images[0], images[1], images[2], images[6]]
    ov_rects = [rects[0] + [[180.0, 150.0, 280.0, 260.0, 0.8]], [[-2.0, -2.0, 3.0, 3.0, 0.9]], [],
                [[-30.0, 20.0, 40.0, 90.0, 0.9], [30.0, -25.0, 90.0, 50.0, 0.8]]]
    m.dense_chunk_bytes = 2 * 3 * 4 * synthetic.NVER
    ov_b, ov_s = m.overlay_images(ov_images, rects=ov_rects, connectivity=synthetic.make_render_topology().T)
    torch.cuda.synchronize()
    m._engine(torch.device('cuda', 0)).raise_if_error()
    print('sanitizer frames done:', tuple(loc.shape), [len(b) for b in boxes], [len(b) for b in big], [len(t[0]) for t in out])
    print('sanitizer images done:', [tuple(x.shape) for x in loc_i], [len(b) for b in boxes_i], [len(t[0]) for t in out_i])
    print('sanitizer overlay images done:', [x.shape for x in ov_s])


if __name__ == '__main__':
    main()
