"""The FaceBoxes detector on the H100 (SURVEY.md section 8 row f3) against the vectors recorded from the reference's own
network class (seeded synthetic checkpoint, tests/golden/make_golden_render.py) and against the CPU oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import render_port as rp
from synergynet_b200 import _lib, detect, faceboxes, synthetic

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'render_vectors.npz')
TOL = 1e-4      # max|new - ref| / max|ref|, the bar of the main path (fp32 FMA accumulation measures ~1e-6)


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLD, allow_pickle=False))


@pytest.fixture(scope='module')
def sd():
    return synthetic.make_faceboxes_state_dict(0)


@pytest.fixture(scope='module')
def net(sd):
    return faceboxes.FaceBoxesNet(sd, torch.device('cuda', 0))


def _max_rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize('hw', [(250, 333, 0), (120, 96, 1)])
def test_network_outputs_match_reference(gold, net, hw):
    h, w, seed = hw
    img = torch.from_numpy(synthetic.make_scene_u8(h, w, seed)).cuda()
    n0 = net.launch_count
    loc, conf = net.forward(img)
    assert net.launch_count - n0 == 39                                   # 33 convolutions, 2 + 3 pools, softmax: all ours
    assert _max_rel(loc.cpu().numpy(), gold[f'fbs_loc_{h}x{w}']) <= TOL
    assert _max_rel(conf.cpu().numpy(), gold[f'fbs_conf_{h}x{w}']) <= TOL
    assert np.allclose(conf.sum(1).cpu().numpy(), 1.0, atol=1e-6)


def test_odd_sizes_against_oracle(sd, net):
    for (h, w, seed) in ((33, 47, 2), (200, 129, 3), (64, 64, 4)):
        scene = synthetic.make_scene_u8(h, w, seed)
        loc, conf = net.forward(torch.from_numpy(scene).cuda())
        l_ref, c_ref = rp.faceboxes_forward(sd, scene)
        assert loc.shape == l_ref.shape == (detect.num_priors(h, w), 4)
        assert _max_rel(loc.cpu().numpy(), l_ref) <= TOL and _max_rel(conf.cpu().numpy(), c_ref) <= TOL


def test_detector_chain_is_exact_given_the_network_outputs(net):
    """Decode + ordering + NMS on the device against the oracle's post-processing of the SAME loc / conf: index lists
    identical, boxes to the exp() tolerance."""
    scene = synthetic.make_scene_u8(250, 333, 0)
    loc, conf = net.forward(torch.from_numpy(scene).cuda())
    dets, n = detect.decode_device(loc, conf, 250, 333)
    n = int(n.item())
    want = rp.faceboxes_dets(loc.cpu().numpy(), conf.cpu().numpy(), 250, 333)
    got = dets[:n].cpu().numpy()
    assert got.shape == want.shape and np.array_equal(got[:, 4], want[:, 4])
    assert np.allclose(got[:, :4], want[:, :4], rtol=2e-6, atol=2e-5)
    keep, nk = detect.nms_device(dets, 0.3, _lib.NMS_CPU_NMS, n=n)
    assert keep[:int(nk.item())].cpu().numpy().tolist() == rp.cpu_nms(got, 0.3)


def _match_fraction(got, want, tol=0.05):
    """Fraction of the reference's boxes that have a detection with the same score (1e-4) and corners within `tol` pixels."""
    if want.shape[0] == 0:
        return 1.0 if got.shape[0] == 0 else 0.0
    hit = 0
    for b in want:
        d = np.abs(got[:, 4] - b[4]) < 1e-4 * max(abs(b[4]), 1e-3)
        hit += bool(d.any() and (np.abs(got[d][:, :4] - b[:4]).max(1) < tol).any())
    return hit / want.shape[0]


def test_reference_shaped_detector(gold, sd):
    """``FaceBoxes(...)(img)`` end to end against what the reference's FaceBoxes.__call__ returned.  NMS decisions are
    discontinuous in the boxes, so a box pair whose overlap sits within float noise of the threshold may flip: nearly
    all boxes must coincide, not every one."""
    fb = faceboxes.FaceBoxes(weights=sd, device='cuda:0')
    for (h, w, seed) in ((250, 333, 0), (120, 96, 1)):
        got = np.array(fb(synthetic.make_scene_u8(h, w, seed)), np.float32).reshape(-1, 5)
        want = gold[f'fbs_final_{h}x{w}']
        assert abs(got.shape[0] - want.shape[0]) <= max(2, want.shape[0] // 50)
        assert _match_fraction(got, want) >= 0.97
        assert (got[:, 4] > detect.vis_thres).all() and (np.diff(got[:, 4]) <= 0).all()


def test_oversized_image_is_rescaled_like_the_reference(sd):
    """FaceBoxes.py:62-79: images above 720 x 1080 are shrunk with cv2.resize on the host, boxes divided by the scale."""
    import cv2
    scene = synthetic.make_scene_u8(900, 1300, 5)
    fb = faceboxes.FaceBoxes(weights=sd, device='cuda:0')
    got = np.array(fb(scene), np.float32).reshape(-1, 5)
    scale = 720 / 900
    if 1300 * scale > 1080:
        scale *= 1080 / (1300 * scale)
    small = cv2.resize(scene, dsize=(int(scale * 1300), int(scale * 900)))
    loc, conf = rp.faceboxes_forward(sd, small)
    d = rp.faceboxes_dets(loc, conf, small.shape[0], small.shape[1], scale=scale)
    want = d[rp.cpu_nms(d, 0.3)][:750]
    want = want[want[:, 4] > 0.5]
    assert abs(got.shape[0] - want.shape[0]) <= max(2, want.shape[0] // 50) and _match_fraction(got, want, tol=0.1) >= 0.97


def test_state_errors():
    lib = _lib.load()
    import ctypes as C
    h = C.c_void_p()
    _lib.check(lib.syn_fb_create(0, C.byref(h)))
    assert lib.syn_fb_commit(h) == 3                                      # SYN_ERR_STATE: layers never set
    one = torch.zeros(8, device='cuda')
    assert lib.syn_fb_forward(h, one.data_ptr(), 64, 64, one.data_ptr(), one.data_ptr(), None) == 3
    w = torch.zeros(10)
    assert lib.syn_fb_set_layer(h, 0, w.data_ptr(), 10, None, w.data_ptr(), w.data_ptr(), w.data_ptr(), w.data_ptr(), 1e-5) == 4
    lib.syn_fb_destroy(h)
