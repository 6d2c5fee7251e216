"""The crop + resize kernel on the device against the host path it replaces (crop_img + cv2.resize) and against the cv2
digests committed in tests/golden/resize_digests.json, in both output layouts; and get_all_outputs fed by it."""
import json
import os
import types

import numpy as np
import pytest
import torch

from golden import make_golden_resize as gr
from oracle import synth_model
from synergynet_b200 import faceboxes, synthetic
from synergynet_b200.inference import INTER_LANCZOS4, INTER_LINEAR, crop_resize_device, roi_affine, square_roi

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def gold():
    with open(os.path.join(HERE, 'golden', 'resize_digests.json')) as f:
        return json.load(f)


@pytest.fixture(scope='module')
def scene():
    return synthetic.make_scene_u8(*gr.SCENE)


@pytest.mark.parametrize('name', list(gr.MODES))
def test_face_crops_match_host_path_and_digests(scene, gold, name):
    mode = gr.MODES[name]
    img = torch.from_numpy(scene).to(DEV)
    planar = crop_resize_device(img, gr.ROIS, (120, 120), mode).cpu().numpy()
    inter = crop_resize_device(img, gr.ROIS, (120, 120), mode, planar=False).cpu().numpy()
    assert planar.shape == (len(gr.ROIS), 3, 120, 120) and inter.shape == (len(gr.ROIS), 120, 120, 3)
    for b, box in enumerate(gr.ROIS):
        want = cv2.resize(gr.host_crop(scene, box), dsize=(120, 120), interpolation=mode)
        assert np.array_equal(inter[b], want), (box, name)
        assert np.array_equal(planar[b], want.transpose(2, 0, 1)), (box, name)
    assert [gr.digest(c) for c in inter] == gold['crops'][name]


def test_non_square_outputs_and_random_boxes(scene):
    """Output sizes other than 120 x 120 and random boxes (partly outside, half-integer corners)."""
    rng = np.random.default_rng(5)
    c = rng.uniform(-40, [1120, 760], (24, 2))
    half = rng.uniform(1, 260, (24, 2))
    boxes = [list(np.round(np.r_[c[i] - half[i], c[i] + half[i]] * 2) / 2) for i in range(24)]
    img = torch.from_numpy(scene).to(DEV)
    for mode in (INTER_LINEAR, INTER_LANCZOS4):
        for (w, h) in ((120, 120), (97, 64), (33, 150)):
            got = crop_resize_device(img, boxes, (w, h), mode, planar=False).cpu().numpy()
            for b, box in enumerate(boxes):
                assert np.array_equal(got[b], cv2.resize(gr.host_crop(scene, box), dsize=(w, h), interpolation=mode)), (box, mode, w, h)


def test_detector_shrinks_match_cv2(gold):
    for k, (h, w) in enumerate(gr.SHRINKS):
        img = synthetic.make_scene_u8(h, w, k)
        hs, ws = gr.detector_size(h, w)
        got = crop_resize_device(torch.from_numpy(img).to(DEV), [[0, 0, w, h]], (ws, hs), INTER_LINEAR, planar=False)[0].cpu().numpy()
        assert np.array_equal(got, cv2.resize(img, dsize=(ws, hs))), (h, w)
        assert gr.digest(got) == gold['shrinks'][f'{h}x{w}']


@pytest.mark.parametrize('hw', [(900, 1300), (1440, 2160)])
def test_faceboxes_network_sees_the_cv2_shrink(hw):
    """FaceBoxes.__call__ on an oversized image hands its network the bytes cv2.resize makes on the host."""
    det = faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0), device='cuda:0')
    seen = []
    forward = det.net.forward
    det.net.forward = lambda image: (seen.append(image.cpu().numpy()), forward(image))[1]
    scene = synthetic.make_scene_u8(*hw, 2)
    det(scene)
    hs, ws = gr.detector_size(*hw)
    assert len(seen) == 1 and np.array_equal(seen[0], cv2.resize(scene, dsize=(ws, hs)))


@pytest.fixture(scope='module')
def model(synth_pack):
    from synergynet_b200 import model_building
    m = model_building.SynergyNet(types.SimpleNamespace(arch='mobilenet_v2', img_size=120, devices_id=[0]))
    m.load_state_dict(synth_model.build_state_dict(0), strict=True)
    m.eval()
    return m


@pytest.mark.parametrize('interp', ['lanczos4', 'linear'])
def test_get_all_outputs_equals_host_made_crops(model, interp):
    """get_all_outputs on a 16-face scene returns exactly what forward_landmarks + the image-space stages give for the
    crops crop_img + cv2.resize make on the host."""
    scene = synthetic.make_scene_u8(720, 1080, 9)
    rng = np.random.default_rng(1)
    xy = rng.uniform([-30, -30], [1000, 640], (16, 2))
    side = rng.uniform(60, 330, 16)
    rects = [[float(x), float(y), float(x + s * 0.8), float(y + s), 0.9] for (x, y), s in zip(xy, side)]
    old = model.resize_interpolation
    model.resize_interpolation = interp
    try:
        lmk, mesh, pose = model.get_all_outputs(scene.copy(), rects=rects)
    finally:
        model.resize_interpolation = old
    mode = INTER_LANCZOS4 if interp == 'lanczos4' else INTER_LINEAR
    boxes = [square_roi(list(r)) for r in rects]
    crops = np.stack([cv2.resize(gr.host_crop(scene, b), dsize=(120, 120), interpolation=mode) for b in boxes])
    eng = model._engine(DEV)
    _, params = eng.forward_landmarks(torch.from_numpy(crops).permute(0, 3, 1, 2).contiguous().to(DEV), want_params=True)
    roi5 = torch.from_numpy(roi_affine(boxes)).to(DEV)
    want_lmk = eng.reconstruct_image(params, roi5, dense=False).cpu().numpy()
    want_mesh = eng.reconstruct_image(params, roi5, dense=True).cpu().numpy()
    ang, t3d = eng.pose_decode(params, roi5)
    assert np.array_equal(np.stack(lmk), want_lmk) and np.array_equal(np.stack(mesh), want_mesh)
    assert [p[0] for p in pose] == ang.cpu().numpy().tolist()
    assert np.array_equal(np.stack([p[1] for p in pose]), t3d.cpu().numpy())
