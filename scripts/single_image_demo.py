#!/usr/bin/env python
"""The reference's single-image flow (singleImage.py:20-75, utils/render.py:31-53) on the H100 modules: detect faces,
regress 3DMM parameters, reconstruct landmarks / dense meshes / poses, draw the solid-mesh overlay.

    python scripts/single_image_demo.py [image.png] [--out overlay.png]

Without an image a synthetic scene is used; without the reference's external assets (pretrained/best.pth.tar,
3dmm_data/, FaceBoxes/weights/FaceBoxesProd.pth) the seeded synthetic stand-ins of synergynet_b200.synthetic are used, so
the picture is meaningless but every stage runs exactly as it would with the real files.  Needs an H100."""
import argparse
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('image', nargs='?')
    ap.add_argument('--out', default='demo_overlay.png')
    ap.add_argument('--max-faces', type=int, default=8)
    ap.add_argument('--detector-weights', default=None, help='FaceBoxesProd.pth of the reference; default: synthetic weights')
    ap.add_argument('--checkpoint', default=None, help='pretrained/best.pth.tar of the reference; default: synthetic weights')
    args = ap.parse_args()
    import cv2
    from synergynet_b200 import Sim3DR, faceboxes, model_building, synthetic
    from synergynet_b200.params import ParamsPack, set_param_pack

    img = cv2.imread(args.image) if args.image else synthetic.make_scene_u8(480, 640, 0)
    if os.environ.get('SYNERGY_3DMM_DIR') is None:
        set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))
    model = model_building.SynergyNet(types.SimpleNamespace(arch='mobilenet_v2', img_size=120, devices_id=[0]))
    if args.checkpoint:
        model.load_weights(args.checkpoint)
    else:
        synthetic.seeded_init_(model, 0)                     # random-init weights of the reference architecture, as bench.py uses
        synthetic.randomize_batchnorm_(model, 0)
    model.eval()
    det = faceboxes.FaceBoxes(weights=args.detector_weights or synthetic.make_faceboxes_state_dict(0))
    model.face_detector = lambda im: det(im)[:args.max_faces]
    lmks, meshes, poses = model.get_all_outputs(img)         # synergy3DMM.py:167-207, every stage on the GPU
    print(f'{len(lmks)} faces; first pose (yaw, pitch, roll) = {poses[0][0] if poses else None}')
    tri = model.triangles.cpu().numpy().T.astype(np.int32) if args.checkpoint else synthetic.make_render_topology()
    blended, overlap = Sim3DR.render(img, meshes, np.ascontiguousarray(tri), alpha=0.6, wfp=args.out)
    print('wrote', args.out, 'and', args.out[:-4] + '_solid.png')


if __name__ == '__main__':
    main()
