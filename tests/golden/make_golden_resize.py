"""Digests of crops and detector shrinks made by cv2 (crop_img + cv2.resize), the bytes the device crop + resize must
reproduce.  The get_all_outputs goldens were recorded from crops this OpenCV build made; pinning its resize output here
lets a test on another machine show that its cv2 (the host path the GPU tests compare with) makes the same bytes.

    python tests/golden/make_golden_resize.py        # writes tests/golden/resize_digests.json

The cases are defined here and imported by tests/test_resize_emulation.py and tests/test_gpu_crop.py.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, 'resize_digests.json')

SCENE = (720, 1080, 3)           # synthetic.make_scene_u8(720, 1080, 3): the image every ROI is cut from

# ROI boxes as get_all_outputs passes them to crop_img: float x0, y0, x1, y1 (rounded half-even there)
ROIS = (
    # square, inside the image, sides around the 120 output and the exact halving (240)
    [[300 + s % 7, 200 + s % 5, 300 + s % 7 + s, 200 + s % 5 + s] for s in (1, 2, 7, 60, 100, 119, 120, 121, 200, 239, 240, 241, 400, 480, 520)]
    # non-square
    + [[50, 60, 140, 190], [400, 100, 700, 270], [900, 10, 917, 250], [10, 600, 250, 607], [600, 300, 1080, 540]]
    # partly outside (zero fill, replicated by the resampler's border), including a halving and a 1-pixel overlap
    + [[-30, -20, 90, 100], [1000, 600, 1160, 760], [-50, 300, 190, 540], [700, -239, 940, 1], [-399, 700, 1, 740],
       [1079, 719, 1200, 840]]
    # wholly outside
    + [[1100, 100, 1200, 200], [-300, -300, -60, -60], [200, 730, 440, 970]]
    # fractional boxes: round-half-even decides the integer crop (10.5 -> 10, 11.5 -> 12)
    + [[10.5, 11.5, 250.5, 251.5], [33.49, 40.51, 150.2, 157.7], [500.5, 300.5, 620.5, 420.5], [-12.5, 30.5, 107.5, 150.5]]
)
MODES = {'linear': 1, 'lanczos4': 4}
# FaceBoxes.__call__ inputs above 720 x 1080 (H, W): each shrinks to int(scale*h) x int(scale*w), INTER_LINEAR
SHRINKS = [(900, 1300), (1080, 1920), (2160, 3840), (1440, 2160), (1000, 1000), (721, 1080)]


def detector_size(h, w):
    """FaceBoxes/FaceBoxes.py:62-79: (h_s, w_s) of the network input."""
    scale = 1
    if h > 720:
        scale = 720 / h
    if w * scale > 1080:
        scale *= 1080 / (w * scale)
    return int(scale * h), int(scale * w)


def host_crop(img: np.ndarray, box) -> np.ndarray:
    """crop_img (zero fill outside the image), also for a box wholly outside the image, where crop_img's slicing raises
    and the device crop is all zeros."""
    from synergynet_b200.inference import crop_img, roi_ints
    x0, y0, x1, y1 = roi_ints(box)
    h, w = img.shape[:2]
    if min(x1, w) > max(x0, 0) and min(y1, h) > max(y0, 0):
        return crop_img(img, box)
    return np.zeros((y1 - y0, x1 - x0, 3), np.uint8)


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).hexdigest()


def record():
    import cv2
    from synergynet_b200 import synthetic
    scene = synthetic.make_scene_u8(*SCENE)
    out = {'opencv': cv2.__version__, 'crops': {}, 'shrinks': {}}
    for name, mode in MODES.items():
        out['crops'][name] = [digest(cv2.resize(host_crop(scene, r), dsize=(120, 120), interpolation=mode)) for r in ROIS]
    for k, (h, w) in enumerate(SHRINKS):
        hs, ws = detector_size(h, w)
        out['shrinks'][f'{h}x{w}'] = digest(cv2.resize(synthetic.make_scene_u8(h, w, k), dsize=(ws, hs)))
    return out


if __name__ == '__main__':
    with open(OUT, 'w') as f:
        json.dump(record(), f, indent=1)
        f.write('\n')
    print('wrote', OUT)
