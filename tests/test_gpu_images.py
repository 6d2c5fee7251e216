"""The image-list path on the H100 against the one-image path it mirrors: detector network (every launch), decode, NMS,
crops, ``detect_images`` and ``get_all_outputs_images``, on images of different sizes.  The oracle of a result is the
one-image call on each image, which test_gpu_fb_stages.py / test_gpu_faceboxes.py / test_gpu_crop.py hold to the float64
oracles and the reference's vectors; every equality here is bit for bit."""
import random

import numpy as np
import pytest
import torch

from oracle import fb64, synth_mbv1, synth_model, synth_resnet
from oracle.stage_check import make_model
from synergynet_b200 import _lib, detect, faceboxes, synthetic
from synergynet_b200.inference import (INTER_LANCZOS4, INTER_LINEAR, ImagePack, crop_resize_device, crop_resize_images_device,
                                       pack_images)

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def sd():
    return synthetic.make_faceboxes_state_dict(0)


@pytest.fixture(scope='module')
def net(sd):
    return faceboxes.FaceBoxesNet(sd, DEV)


@pytest.fixture(scope='module')
def fb(sd):
    return faceboxes.FaceBoxes(weights=sd, device='cuda:0')


@pytest.fixture(scope='module')
def synth_pack():
    from synergynet_b200.params import ParamsPack, set_param_pack
    set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))


def _images(sizes, seed=0):
    return [synthetic.make_scene_u8(h, w, seed + 7 * i + h + w) for i, (h, w) in enumerate(sizes)]


def _mixed(seed=0):
    """fb64.choose_sizes() (720 x 1080, 1 x 1, 1 x 333 ...) shuffled with repeats: 64-row tiles straddle frames of different
    sizes, and several 1 x 1 frames share one tile."""
    sizes = fb64.choose_sizes()
    sizes = sizes + [sizes[3], (1, 1), (120, 96)]
    random.Random(seed).shuffle(sizes)
    return sizes


def _dev(images):
    return [torch.from_numpy(np.ascontiguousarray(im)).to(DEV) for im in images]


# ---- the network ---------------------------------------------------------------------------------------------------------
def test_forward_images_equals_forward_per_image(net):
    sizes = _mixed()
    ims = _dev(_images(sizes))
    n0 = net.launch_count
    loc, conf = net.forward_images(ims)
    assert net.launch_count - n0 == 39
    for i, (h, w) in enumerate(sizes):
        l1, c1 = net.forward(ims[i])
        assert loc[i].shape == (detect.num_priors(h, w), 4)
        assert torch.equal(loc[i], l1) and torch.equal(conf[i], c1), f'image {i} {h}x{w}'
    torch.cuda.synchronize()


def test_every_launch_equals_the_one_image_launch(net):
    """All 39 launches: every image's map of a stage equals that stage of the one-image debug run, channel slices that
    later launches write included (both start from a zeroed workspace).  The list is fb64.choose_sizes() shuffled with
    repeats, 720 x 1080 included."""
    sizes = _mixed(seed=5)
    ims = _dev(_images(sizes, seed=5))
    for stage in range(39):
        got = net.debug_forward_images_until(ims, stage)
        for i in range(len(sizes)):
            want = net.debug_forward_until(ims[i], stage)
            assert got[i].shape == want.shape
            assert torch.equal(got[i].view(torch.int32), want.view(torch.int32)), f'stage {stage} image {i} {sizes[i]}'
    torch.cuda.synchronize()


def test_equal_sizes_match_forward_batch_and_the_workspace_grows(sd):
    net = faceboxes.FaceBoxesNet(sd, DEV)
    a = _dev(_images([(120, 96)] * 3, seed=1))
    stack = torch.stack(a)
    small = net.forward_images(a)
    big = net.forward_images(_dev(_images([(720, 1080), (1, 1)], seed=2)))
    again = net.forward_images(a)
    lb, cb = net.forward_batch(stack)
    torch.cuda.synchronize()
    for i in range(3):
        assert torch.equal(small[0][i], lb[i]) and torch.equal(small[1][i], cb[i])
        assert torch.equal(again[0][i], lb[i]) and torch.equal(again[1][i], cb[i])
    one = _dev(_images([(720, 1080), (1, 1)], seed=2))[1]
    assert torch.equal(big[0][1], net.forward(one)[0]) and torch.equal(big[1][1], net.forward(one)[1])
    net.close()


# ---- decode and NMS ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', [_lib.NMS_CPU_NMS, _lib.NMS_PY_CPU_NMS])
def test_decode_and_nms_equal_the_one_image_calls(net, mode):
    sizes = [(250, 333), (1, 1), (720, 1080), (120, 96), (33, 993)]
    ims = _dev(_images(sizes, seed=9))
    loc, conf, p = net.forward_packed(ims)
    scales = [1.0, 0.5, 0.75, 1.0, 0.3]
    dets, n = detect.decode_images_device(loc, conf, sizes, scales)
    keep, n_keep = detect.nms_batch_device(dets, n, detect.nms_threshold, mode)
    assert dets.shape == (5, min(detect.top_k, max(detect.num_priors(h, w) for h, w in sizes)), 5)
    for i, (h, w) in enumerate(sizes):
        d1, n1 = detect.decode_device(loc[p[i]:p[i + 1]], conf[p[i]:p[i + 1]], h, w, scale=scales[i])
        c = int(n1.item())
        assert int(n[i].item()) == c
        assert torch.equal(dets[i, :c], d1[:c]), f'image {i}'
        k1, nk1 = detect.nms_device(d1, detect.nms_threshold, mode, n=c)
        assert int(n_keep[i].item()) == int(nk1.item())
        assert torch.equal(keep[i, :int(nk1.item())], k1[:int(nk1.item())]), f'image {i}'


# ---- crops ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', [INTER_LANCZOS4, INTER_LINEAR])
def test_crops_equal_the_one_image_crops(mode):
    sizes = [(250, 333), (1, 1), (97, 61), (720, 1080)]
    host = _images(sizes, seed=11)
    pack = pack_images(host, DEV)
    rois = [[-30.4, -12.0, 80.6, 99.5], [10.0, 10.0, 200.0, 150.0], [-3.0, -3.0, 4.0, 5.0], [20.0, 30.0, 60.0, 90.0],
            [500.0, 600.0, 1200.0, 760.0], [-1.0, -1.0, 2.0, 2.0]]
    idx = [0, 0, 1, 2, 3, 1]
    got = crop_resize_images_device(pack, idx, rois, (120, 120), mode)
    per = [(33, 17), (120, 120), (5, 9), (64, 3), (1, 1), (200, 150)]
    flat = crop_resize_images_device(pack, idx, rois, per, mode, planar=False)
    at = 0
    for b in range(len(rois)):
        image = torch.from_numpy(host[idx[b]]).to(DEV)
        assert torch.equal(got[b], crop_resize_device(image, [rois[b]], (120, 120), mode)[0]), f'ROI {b}'
        w, h = per[b]
        one = crop_resize_device(image, [rois[b]], (w, h), mode, planar=False)[0]
        assert torch.equal(flat[at:at + 3 * w * h].view(h, w, 3), one), f'ROI {b} at {w}x{h}'
        at += 3 * w * h
    assert at == flat.numel()


# ---- detect_images -------------------------------------------------------------------------------------------------------
def _detect_sizes(n, seed):
    mix = [(250, 333), (1080, 1920), (1500, 900), (120, 96), (1, 1), (721, 1000), (480, 640)]
    rng = random.Random(seed)
    return [mix[i % len(mix)] if i < len(mix) else rng.choice(mix) for i in range(n)]


@pytest.mark.parametrize('n', [1, 65, 130])
def test_detect_images_equals_call_per_image(fb, n):
    sizes = _detect_sizes(n, n)
    host = _images(sizes, seed=n)
    got = fb.detect_images(host)
    assert len(got) == n
    assert got == [fb(im) for im in host]
    if n == 1:
        assert fb.detect_images(_dev(host)) == got                                 # CUDA tensors in


def test_detect_images_on_equal_sizes_equals_detect_batch(fb):
    frames = _images([(360, 480)] * 5, seed=3)
    assert fb.detect_images(frames) == fb.detect_batch(np.stack(frames))
    big = _images([(900, 1400)] * 3, seed=4)
    assert fb.detect_images(big) == fb.detect_batch(np.stack(big))


# ---- get_all_outputs_images ----------------------------------------------------------------------------------------------
def _same_outputs(got, want, where):
    (lg, mg, pg), (lw, mw, pw) = got, want
    assert len(lg) == len(mg) == len(pg) == len(lw) == len(mw) == len(pw), where
    for j in range(len(lw)):
        assert np.array_equal(lg[j], lw[j]) and np.array_equal(mg[j], mw[j]), f'{where} face {j}'
        assert pg[j][0] == pw[j][0] and np.array_equal(pg[j][1], pw[j][1]), f'{where} face {j}'


def _checkpoint(arch):
    if arch == 'mobilenet_v2':
        return make_model(synth_model.build_state_dict(0))
    if arch.startswith('resnet'):
        return make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
    return make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)


RECTS = [[[-10.0, -5.0, 50.0, 55.0, 0.9], [150.0, 120.0, 300.0, 230.0, 0.8]], [], [[40.0, 20.0, 100.0, 80.0, 0.7]],
         [[1.0, 1.0, 30.0, 40.0, 0.6], [200.0, 100.0, 600.0, 500.0, 0.9], [-40.0, 300.0, 90.0, 420.0, 0.9]], []]


@pytest.mark.parametrize('arch', ['mobilenet_v2', 'resnet18', 'mobilenet_05'])
def test_get_all_outputs_images_equals_get_all_outputs(synth_pack, fb, arch):
    model = _checkpoint(arch)
    eng = model._engine(DEV)
    sizes = [(360, 480), (1, 1), (250, 333), (720, 1080), (97, 61)]
    images = _images(sizes, seed=21)
    got = model.get_all_outputs_images(images, rects=RECTS)
    assert [len(t[0]) for t in got] == [2, 0, 1, 3, 0] and got[1] == ([], [], []) and got[4] == ([], [], [])
    for i in range(len(sizes)):
        _same_outputs(got[i], model.get_all_outputs(images[i].copy(), rects=RECTS[i]), f'{arch} image {i}')
    assert model.get_all_outputs_images(images, rects=[[]] * 5) == [([], [], [])] * 5
    model.face_detector = fb
    try:
        small = _images([(240, 320), (300, 200), (1100, 1500)], seed=6 - 560)
        auto = model.get_all_outputs_images(small)
        rects = fb.detect_images(small)
        for i in range(3):
            _same_outputs(auto[i], model.get_all_outputs(small[i].copy(), rects=rects[i]), f'{arch} detected image {i}')
        model.face_detector = lambda im: fb(im)[:2]                                # no detect_images: image by image
        per = model.get_all_outputs_images(small)
        assert [len(t[0]) for t in per] == [min(2, len(r)) for r in rects]
    finally:
        model.face_detector = None
    assert eng.poll_error() == 0 and eng.poll_saturation(warn=False) == 0


# ---- errors leave the device usable --------------------------------------------------------------------------------------
def test_errors_leave_the_device_usable(net, fb):
    ims = _dev(_images([(120, 96), (33, 61)]))
    good = net.forward_images(ims)
    with pytest.raises(ValueError, match='at least one image'):
        fb.detect_images([])
    with pytest.raises(ValueError):
        net.forward_images([ims[0].float()])
    with pytest.raises(ValueError):
        net.forward_images([ims[0][:, ::2]])                                       # not contiguous
    with pytest.raises(ValueError):
        net.forward_images([ims[0].cpu()])                                         # wrong device
    with pytest.raises(ValueError, match='1..64'):
        net.forward_images([ims[1]] * 65)
    with pytest.raises(ValueError, match='outside 0..38'):
        net.debug_forward_images_until(ims, 39)
    lib = _lib.load()
    hs, ws = np.array([120, 0], np.int32), np.array([96, 61], np.int32)
    loc = torch.empty((4096, 4), device=DEV)
    conf = torch.empty((4096, 2), device=DEV)
    n0 = net.launch_count
    assert lib.syn_fb_forward_images(net._h, ims[0].data_ptr(), 2, hs.ctypes.data, ws.ctypes.data, loc.data_ptr(), conf.data_ptr(), None) == 1
    assert b'image 1 is 0x61' in lib.syn_last_error()
    big = np.full(_lib.FB_MAX_FRAMES + 1, 33, np.int32)
    assert lib.syn_fb_forward_images(net._h, ims[0].data_ptr(), _lib.FB_MAX_FRAMES + 1, big.ctypes.data, big.ctypes.data,
                                     loc.data_ptr(), conf.data_ptr(), None) == 1
    assert b'65 frames, 1..64 per call' in lib.syn_last_error()
    # packed images on another device: the network refuses them, detect_images moves them to the detector's device
    host_pack = pack_images(_images([(120, 96), (33, 61)]), 'cpu')
    with pytest.raises(ValueError, match='detector device'):
        net.forward_packed(host_pack)
    with pytest.raises(ValueError, match='detector device'):
        net.forward_packed(ImagePack(torch.zeros(3, dtype=torch.float32, device=DEV), [(1, 1)]))        # not uint8
    assert net.launch_count == n0
    assert fb.detect_images(host_pack) == [fb(im) for im in _images([(120, 96), (33, 61)])]
    again = net.forward_images(ims)
    torch.cuda.synchronize()
    for i in range(2):
        assert torch.equal(again[0][i], good[0][i]) and torch.equal(again[1][i], good[1][i])
