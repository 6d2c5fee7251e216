"""The reference's single-image flow (singleImage.py / utils/render.py) through the H100 modules end to end: detector ->
crops -> backbone -> landmarks, dense meshes, poses -> solid-mesh overlay, every stage on the device and chained without
host copies where the reference hands numpy arrays around."""
import types

import numpy as np
import pytest
import torch

from oracle import render_port as rp
from oracle import synth_model
from synergynet_b200 import Sim3DR, faceboxes, synthetic
from synergynet_b200.inference import RENDER_CFG, roi_affine, square_roi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def model(synth_pack):
    from synergynet_b200 import model_building
    m = model_building.SynergyNet(types.SimpleNamespace(arch='mobilenet_v2', img_size=120, devices_id=[0]))
    m.load_state_dict(synth_model.build_state_dict(0), strict=True)
    m.eval()
    return m


def test_detector_feeds_get_all_outputs(model):
    img = synthetic.make_scene_u8(240, 320, 6)
    det = faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0), device='cuda:0')
    rects = det(img)
    assert len(rects) > 4
    rects = rects[:6]
    model.face_detector = lambda im: det(im)[:6]
    try:
        lmk_a, mesh_a, pose_a = model.get_all_outputs(img.copy())                      # synergy3DMM.py:167-207 with the GPU detector
    finally:
        model.face_detector = None
    lmk_b, mesh_b, pose_b = model.get_all_outputs(img.copy(), rects=rects)
    assert len(lmk_a) == len(rects) == 6
    assert np.array_equal(np.stack(lmk_a), np.stack(lmk_b)) and np.array_equal(np.stack(mesh_a), np.stack(mesh_b))
    assert mesh_a[0].shape == (3, synthetic.NVER) and np.isfinite(np.stack(mesh_a)).all()


def test_dense_meshes_render_without_leaving_the_device(model):
    """Dense vertices stay on the GPU as (B,3,N) and are rendered in place; the same meshes pulled to the host and drawn
    by the oracle (the reference's algorithm) give the same picture: identical uint8 image when fed the same colours."""
    dev = torch.device('cuda', 0)
    img = synthetic.make_scene_u8(240, 320, 6)
    rects = [[40.0, 30.0, 150.0, 160.0, 0.9], [170.0, 70.0, 300.0, 220.0, 0.8]]
    boxes = [square_roi(list(r)) for r in rects]
    import cv2
    from synergynet_b200.inference import crop_img
    crops = np.stack([cv2.resize(crop_img(img, b), dsize=(120, 120), interpolation=cv2.INTER_LINEAR) for b in boxes])
    eng = model._engine(dev)
    _, params = eng.forward_landmarks(torch.from_numpy(crops).permute(0, 3, 1, 2).contiguous().to(dev), want_params=True)
    dense = eng.reconstruct_image(params, torch.from_numpy(roi_affine(boxes)).to(dev), dense=True)     # (2,3,53215) on the device
    assert dense.is_cuda and tuple(dense.shape) == (2, 3, synthetic.NVER)
    # the synthetic 3DMM has no meaningful surface: draw a subset of the grid topology (any triangle list is a valid input)
    tri = np.ascontiguousarray(synthetic.make_render_topology()[::97][:900])
    r = Sim3DR.MeshRenderer(tri, synthetic.NVER, dev)
    v = dense.transpose(1, 2)                                                         # strided view of the kernel's output
    nrm = r.normals(v)
    col = r.colors(v, nrm, Sim3DR._light_cfg(**RENDER_CFG))
    canvas = torch.from_numpy(img.copy()).to(dev)
    r.rasterize(canvas, v, col)
    host = dense.cpu().numpy()
    want = img.copy()
    for b in range(2):
        vb = np.ascontiguousarray(host[b].T)
        n_ref = rp.get_normal(vb, tri)
        used = np.unique(tri)
        assert np.array_equal(nrm[b].cpu().numpy()[used], n_ref[used])
        want = rp.rasterize(vb, tri, col[b].cpu().numpy(), want)
    assert np.array_equal(canvas.cpu().numpy(), want)
    assert (want != img).any()
    blended, overlap = Sim3DR.render(img, [host[0], host[1]], tri)                    # utils/render.py:31-53, batched
    assert np.array_equal(overlap, want) and blended.dtype == np.uint8
