#!/usr/bin/env python
"""scripts/single_image_demo.py for a batch of frames: a seeded stack of synthetic scenes goes through
``get_all_outputs_batch`` (one detector pass, one crop launch, one backbone call for the faces of all frames) and every
frame gets its solid-mesh overlay.

    python scripts/frames_demo.py [--frames 4] [--out-dir frames_demo]

The seeded synthetic stand-ins of synergynet_b200.synthetic replace the reference's external assets, so the pictures are
meaningless but every stage runs as it would with the real files.  Needs an H100."""
import argparse
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _TopFaces:
    """The detector, keeping the ``max_faces`` best boxes of every frame."""

    def __init__(self, det, max_faces):
        self.det, self.max_faces = det, max_faces

    def detect_batch(self, frames):
        return [r[:self.max_faces] for r in self.det.detect_batch(frames)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=4)
    ap.add_argument('--height', type=int, default=480)
    ap.add_argument('--width', type=int, default=640)
    ap.add_argument('--max-faces', type=int, default=8)
    ap.add_argument('--out-dir', default='frames_demo')
    args = ap.parse_args()
    from synergynet_b200 import Sim3DR, faceboxes, model_building, synthetic
    from synergynet_b200.params import ParamsPack, set_param_pack

    frames = np.stack([synthetic.make_scene_u8(args.height, args.width, seed) for seed in range(args.frames)])
    set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))
    model = model_building.SynergyNet(types.SimpleNamespace(arch='mobilenet_v2', img_size=120, devices_id=[0]))
    synthetic.seeded_init_(model, 0)
    synthetic.randomize_batchnorm_(model, 0)
    model.eval()
    model.face_detector = _TopFaces(faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0)), args.max_faces)
    results = model.get_all_outputs_batch(frames)
    tri = np.ascontiguousarray(synthetic.make_render_topology())
    os.makedirs(args.out_dir, exist_ok=True)
    for i, (lmks, meshes, poses) in enumerate(results):
        out = os.path.join(args.out_dir, f'frame{i:03d}.png')
        if meshes:
            Sim3DR.render(frames[i], meshes, tri, alpha=0.6, wfp=out)                 # batched over the frame's meshes
        print(f'frame {i}: {len(lmks)} faces' + (f', first pose {poses[0][0]}, wrote {out}' if meshes else ''))


if __name__ == '__main__':
    main()
