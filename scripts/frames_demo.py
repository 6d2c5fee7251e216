#!/usr/bin/env python
"""scripts/single_image_demo.py for a batch of frames: a seeded stack of synthetic scenes goes through
``overlay_batch`` (one detector pass, one crop launch, one backbone call for the faces of all frames, then every face's
dense mesh lit, drawn and blended onto its frame on the device) and each frame's overlay is written as one image.

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
    import cv2
    from synergynet_b200 import faceboxes, model_building, synthetic
    from synergynet_b200.params import ParamsPack, set_param_pack

    frames = np.stack([synthetic.make_scene_u8(args.height, args.width, seed) for seed in range(args.frames)])
    set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))
    model = model_building.SynergyNet(types.SimpleNamespace(arch='mobilenet_v2', img_size=120, devices_id=[0]))
    synthetic.seeded_init_(model, 0)
    synthetic.randomize_batchnorm_(model, 0)
    model.eval()
    model.face_detector = _TopFaces(faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0)), args.max_faces)
    # one pass for the whole stack: detector, crops, backbone, dense meshes, lighting, z-buffer and blend on the device
    blended, _solid = model.overlay_batch(frames, alpha=0.6, connectivity=synthetic.make_render_topology().T)
    os.makedirs(args.out_dir, exist_ok=True)
    for i in range(len(frames)):
        out = os.path.join(args.out_dir, f'frame{i:03d}.png')
        cv2.imwrite(out, blended[i])
        print(f'frame {i}: {int((blended[i] != frames[i]).any(-1).sum())} pixels overlaid, wrote {out}')

if __name__ == '__main__':
    main()
