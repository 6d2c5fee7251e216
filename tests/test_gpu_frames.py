"""The frame-batch path on the H100 against the one-image path it mirrors: detector network (every launch), decode, NMS,
cross-frame crops, ``detect_batch`` and ``get_all_outputs_batch``.  The oracle of a batched result is the one-image call
on each frame, which test_gpu_fb_stages.py / test_gpu_faceboxes.py / test_gpu_crop.py hold to the float64 oracles and the
reference's vectors; the network, decode, NMS and crops must agree with it bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import synth_mbv1, synth_model, synth_resnet
from oracle.stage_check import make_model
from synergynet_b200 import _lib, detect, faceboxes, synthetic
from synergynet_b200.inference import INTER_LANCZOS4, INTER_LINEAR, crop_resize_device, crop_resize_frames_device

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
# maps whose pixel count is not a multiple of 64 (test_gpu_fb_stages.py's sizes): 64-row tiles straddle two frames, and at
# 1 x 1 / 1 x 333 one tile holds every frame of the batch
ODD = ((771, 258), (33, 993), (193, 961), (1, 333), (1, 1))


@pytest.fixture(scope='module')
def sd():
    return synthetic.make_faceboxes_state_dict(0)


@pytest.fixture(scope='module')
def net(sd):
    return faceboxes.FaceBoxesNet(sd, DEV)


@pytest.fixture(scope='module')
def fb(sd):
    return faceboxes.FaceBoxes(weights=sd, device='cuda:0')


def _frames(n, h, w, seed=0):
    """n different seeded scenes of one size, (n,h,w,3) uint8 on the host."""
    return np.stack([synthetic.make_scene_u8(h, w, seed + 13 * i + h + w) for i in range(n)])


def _bits(a, b):
    """Bit equality that also holds where both are NaN."""
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---- 1, 7: the network, bit for bit; 39 launches whatever N ---------------------------------------------------------------
CASES = [(n, h, w) for (h, w) in ((250, 333), (120, 96)) for n in (1, 2, 5)] + [(3, 720, 1080)] + [(3, h, w) for h, w in ODD]


@pytest.mark.parametrize('n,h,w', CASES, ids=[f'{n}x{h}x{w}' for n, h, w in CASES])
def test_forward_batch_equals_forward_per_frame(net, n, h, w):
    frames = _frames(n, h, w)
    assert n == 1 or h * w < 100 or not np.array_equal(frames[0], frames[-1])
    stack = torch.from_numpy(frames).to(DEV)
    n0 = net.launch_count
    loc, conf = net.forward_batch(stack)
    assert net.launch_count - n0 == 39
    p = detect.num_priors(h, w)
    assert tuple(loc.shape) == (n, p, 4) and tuple(conf.shape) == (n, p, 2)
    for i in range(n):
        l1, c1 = net.forward(stack[i])
        assert torch.equal(loc[i], l1) and torch.equal(conf[i], c1), f'frame {i}'
    torch.cuda.synchronize()


def test_a_frame_has_the_same_bits_at_any_index(net):
    h, w = 250, 333
    frames = _frames(5, h, w, seed=3)
    first = torch.from_numpy(frames).to(DEV)
    last = torch.from_numpy(np.ascontiguousarray(frames[::-1])).to(DEV)          # frame 0 now sits at index N - 1
    la, ca = net.forward_batch(first)
    lb, cb = net.forward_batch(last)
    assert torch.equal(la[0], lb[4]) and torch.equal(ca[0], cb[4])
    assert torch.equal(la, lb.flip(0)) and torch.equal(ca, cb.flip(0))
    assert not torch.equal(la[0], la[1])


# ---- 2: every launch, bit for bit ------------------------------------------------------------------------------------------
def test_every_launch_equals_the_one_image_launch(net):
    h, w = 771, 258
    stack = torch.from_numpy(_frames(3, h, w, seed=5)).to(DEV)
    for stage in range(39):
        got = net.debug_forward_batch_until(stack, stage)
        want = torch.stack([net.debug_forward_until(stack[i], stage) for i in range(3)])
        assert got.shape == want.shape, stage
        assert _bits(got, want), f'stage {stage}'
        if 32 <= stage < 37 and stage != 34:                                    # a head is still to run: its slice reads NaN in both
            assert torch.isnan(got).any() and torch.equal(torch.isnan(got), torch.isnan(want)), stage
        else:
            assert not torch.isnan(got).any(), stage


# ---- 3: decode and NMS per frame -------------------------------------------------------------------------------------------
def _crafted(h, w, counts, seed=0):
    """loc / conf for len(counts) frames whose number of priors above the confidence threshold is counts[i]; scores are
    distinct within a frame except for a few exact ties, boxes overlap enough for NMS to suppress many."""
    p = detect.num_priors(h, w)
    g = torch.Generator().manual_seed(seed)
    loc = torch.randn((len(counts), p, 4), generator=g) * torch.tensor([2.0, 2.0, 0.8, 0.8])
    conf = torch.zeros((len(counts), p, 2))
    for i, c in enumerate(counts):
        face = torch.full((p,), 0.01)
        idx = torch.randperm(p, generator=g)[:c]
        sc = 0.06 + 0.93 * torch.rand(c, generator=g)
        if c > 8:
            sc[1], sc[5] = sc[0], sc[4]                                            # ties: the higher prior index goes first
        face[idx] = sc
        conf[i, :, 1] = face
        conf[i, :, 0] = 1 - face
    return loc.to(DEV), conf.to(DEV)


@pytest.mark.parametrize('mode', [_lib.NMS_CPU_NMS, _lib.NMS_PY_CPU_NMS], ids=['cpu_nms', 'py_cpu_nms'])
def test_decode_and_nms_per_frame(mode):
    h, w, k = 250, 333, 300
    counts = [40, 0, 700, 3, 299, 1200, 1]                                         # none, few, > top_k (k = 300), and in between
    loc, conf = _crafted(h, w, counts)
    dets, n = detect.decode_batch_device(loc, conf, h, w, scale=0.8, k=k)
    keep, n_keep = detect.nms_batch_device(dets, n, 0.3, mode)
    assert n.cpu().tolist() == [min(c, k) for c in counts]
    kept_any = 0
    for i, c in enumerate(counts):
        d1, n1 = detect.decode_device(loc[i], conf[i], h, w, scale=0.8, k=k)
        assert int(n1.item()) == min(c, k) and torch.equal(dets[i], d1), f'frame {i}'
        if min(c, k) == 0:
            assert int(n_keep[i].item()) == 0
            continue
        k1, nk1 = detect.nms_device(d1, 0.3, mode, n=int(n1.item()))
        nk = int(nk1.item())
        assert int(n_keep[i].item()) == nk and torch.equal(keep[i, :nk], k1[:nk]), f'frame {i}'
        kept_any += nk < min(c, k)
    assert kept_any >= 3                                                           # NMS suppressed something in the busy frames


def test_decode_caps_rows_at_the_number_of_priors():
    h, w = 64, 64                                                                  # 21 * 4 + 1 + 1 = 86 priors < top_k
    loc, conf = _crafted(h, w, [86, 10])
    dets, n = detect.decode_batch_device(loc, conf, h, w)
    assert tuple(dets.shape) == (2, 86, 5) and n.cpu().tolist() == [86, 10]
    d1, _ = detect.decode_device(loc[0], conf[0], h, w)
    assert torch.equal(dets[0], d1[:86])


# ---- 4: the detector end to end --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n,h,w', [(1, 250, 333), (4, 250, 333), (3, 900, 1300), (2, 720, 1080)])
def test_detect_batch_equals_the_detector_per_frame(fb, n, h, w):
    frames = _frames(n, h, w, seed=7)
    got = fb.detect_batch(list(frames))
    assert len(got) == n
    for i in range(n):
        want = fb(frames[i])
        assert [[float(v) for v in b] for b in got[i]] == [[float(v) for v in b] for b in want], f'frame {i}'
    assert fb.detect_batch(torch.from_numpy(frames).to(DEV)) == got              # the stack a caller already uploaded


def test_detect_batch_splits_a_stack_above_the_limit(fb, monkeypatch):
    frames = _frames(5, 120, 96, seed=9)
    whole = fb.detect_batch(frames)
    monkeypatch.setattr(_lib, 'FB_MAX_FRAMES', 2)                                  # chunks of 2, 2, 1
    assert fb.detect_batch(frames) == whole


# ---- 5: cross-frame crops --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('interp', [INTER_LANCZOS4, INTER_LINEAR], ids=['lanczos4', 'linear'])
def test_cross_frame_crops_equal_the_one_image_crops(interp):
    h, w = 240, 320
    stack = torch.from_numpy(_frames(4, h, w, seed=11)).to(DEV)
    rng = np.random.default_rng(2)
    per_frame = {0: [[-30.4, -12.2, 90.7, 101.5], [250.2, 180.0, 372.6, 300.7]], 1: [],        # over the edges; no ROI at all
                 2: [list(np.r_[c - s, c + s]) for c, s in zip(rng.uniform(0, (w, h), (24, 2)), rng.uniform(8, 90, (24, 1)))],
                 3: [[0, 0, w, h], [100, 60, 340, 300], [10.5, 20.5, 250.5, 260.5]]}            # 2x shrink (area path)
    index = [f for f, r in per_frame.items() for _ in r]
    boxes = [b for r in per_frame.values() for b in r]
    for planar in (False, True):
        got = crop_resize_frames_device(stack, index, boxes, (120, 120), interp, planar=planar)
        want = torch.cat([crop_resize_device(stack[f], r, (120, 120), interp, planar=planar) for f, r in per_frame.items() if r])
        assert got.shape[0] == 29 and torch.equal(got, want)
    order = list(range(len(boxes)))[::-1]                                          # ROIs need not be grouped by frame
    got = crop_resize_frames_device(stack, [index[i] for i in order], [boxes[i] for i in order], (120, 120), interp)
    assert torch.equal(got, want[order])                                           # `want`: the planar crops of the last pass


def test_frame_shrink_equals_the_one_image_shrink():
    stack = torch.from_numpy(_frames(3, 900, 1300, seed=1)).to(DEV)
    got = crop_resize_frames_device(stack, [0, 1, 2], [[0, 0, 1300, 900]] * 3, (1040, 720), INTER_LINEAR, planar=False)
    for i in range(3):
        assert torch.equal(got[i], crop_resize_device(stack[i], [[0, 0, 1300, 900]], (1040, 720), INTER_LINEAR, planar=False)[0])


# ---- 6: get_all_outputs_batch ----------------------------------------------------------------------------------------------
RECTS = [[[60.3, 80.1, 200.9, 250.4, 0.98], [250.2, -20.0, 372.6, 140.7, 0.91], [300.0, 150.0, 470.0, 350.0, 0.9]],
         [[10.0, 12.0, 130.0, 160.0, 0.7]],
         [],
         [[200.0, 100.0, 330.0, 260.0, 0.8], [-15.5, 200.2, 120.1, 371.0, 0.6]],
         []]


def _same_outputs(got, want, where):
    """The triple of one frame against get_all_outputs of that frame: equal counts and order, and equal bits (the faces of
    all frames share one backbone call, and every backbone computes a face from that face's rows alone)."""
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


@pytest.mark.parametrize('arch', ['mobilenet_v2', 'resnet18', 'mobilenet_05'])
def test_get_all_outputs_batch_equals_get_all_outputs_per_frame(synth_pack, fb, arch):
    """Given rects (a frame without a face in the middle and at the end) and with the detector.  The faces of all frames
    go through one backbone call, so a face's tile position differs from the per-frame call's."""
    model = _checkpoint(arch)
    eng = model._engine(DEV)
    frames = _frames(5, 360, 480, seed=17)
    got = model.get_all_outputs_batch(list(frames), rects=RECTS)
    assert [len(t[0]) for t in got] == [3, 1, 0, 2, 0] and got[2] == ([], [], [])
    for i in range(5):
        _same_outputs(got[i], model.get_all_outputs(frames[i].copy(), rects=RECTS[i]), f'{arch} frame {i}')
    assert got[0][1][0].shape == (3, synthetic.NVER)
    assert model.get_all_outputs_batch(frames, rects=[[], [], [], [], []]) == [([], [], [])] * 5
    # dense meshes in chunks of faces: the same arrays
    model.dense_chunk_bytes = 2 * 3 * 4 * synthetic.NVER
    try:
        chunked = model.get_all_outputs_batch(frames, rects=RECTS)
    finally:
        del model.dense_chunk_bytes
    for i in range(5):
        _same_outputs(chunked[i], got[i], f'{arch} chunked frame {i}')
    # with a detector: detect_batch on the shared device stack, then the same stages
    small = _frames(3, 240, 320, seed=6 - 560)                                     # frame 0: the scene of test_gpu_pipeline.py
    model.face_detector = fb
    try:
        auto = model.get_all_outputs_batch(small)
        rects = fb.detect_batch(small)
        assert sum(len(r) for r in rects) > 0
        for i in range(3):
            _same_outputs(auto[i], model.get_all_outputs(small[i].copy(), rects=rects[i]), f'{arch} detected frame {i}')
        model.face_detector = lambda im: fb(im)[:2]                                # a detector without detect_batch: frame by frame
        per = model.get_all_outputs_batch(small)
        assert [len(t[0]) for t in per] == [min(2, len(r)) for r in rects]
    finally:
        model.face_detector = None
    assert eng.poll_error() == 0 and eng.poll_saturation(warn=False) == 0


def test_get_all_outputs_batch_argument_errors(synth_pack):
    model = _checkpoint('mobilenet_v2')
    frames = _frames(2, 120, 160)
    with pytest.raises(RuntimeError, match='no face detector'):
        model.get_all_outputs_batch(frames)
    with pytest.raises(ValueError, match='1 rect lists for 2 frames'):
        model.get_all_outputs_batch(frames, rects=[[]])


# ---- 8: errors leave the device usable -------------------------------------------------------------------------------------
def test_errors_leave_the_device_usable(net, fb):
    h, w = 120, 96
    frames = _frames(2, h, w)
    stack = torch.from_numpy(frames).to(DEV)
    good = net.forward_batch(stack)
    with pytest.raises(ValueError, match='120x96x3, 120x97x3'):
        fb.detect_batch([frames[0], synthetic.make_scene_u8(120, 97, 1)])
    with pytest.raises(ValueError, match='no frames'):
        fb.detect_batch([])
    with pytest.raises(ValueError):
        net.forward_batch(stack.float())                                           # not uint8
    with pytest.raises(ValueError):
        net.forward_batch(stack[:, :, ::2])                                        # not contiguous
    with pytest.raises(ValueError):
        net.forward_batch(stack.cpu())                                             # wrong device
    with pytest.raises(ValueError):
        net.forward_batch(stack[:0])                                               # no frame
    with pytest.raises(ValueError, match='at most 64'):
        net.forward_batch(stack[:1].expand(65, -1, -1, -1).contiguous())
    for stage in (-1, 39):
        with pytest.raises(ValueError, match='outside 0..38'):
            net.debug_forward_batch_until(stack, stage)
    lib = _lib.load()
    p = detect.num_priors(h, w)
    loc, conf = torch.empty((2, p, 4), device=DEV), torch.empty((2, p, 2), device=DEV)
    n0 = net.launch_count
    over = _lib.FB_MAX_FRAMES + 1                                                  # the raw entry refuses before it reads or launches anything
    assert lib.syn_fb_forward_batch(net._h, stack.data_ptr(), over, h, w, loc.data_ptr(), conf.data_ptr(), None) == 1
    assert b'65 frames' in lib.syn_last_error()
    out = torch.empty(8, device=DEV)
    assert lib.syn_fb_debug_forward_batch_until(net._h, stack.data_ptr(), 2, h, w, 39, out.data_ptr(), 8, loc.data_ptr(), conf.data_ptr(), None) == 1
    assert lib.syn_fb_debug_forward_batch_until(net._h, stack.data_ptr(), 2, h, w, 5, out.data_ptr(), 8, loc.data_ptr(), conf.data_ptr(), None) == 4
    fresh = C.c_void_p()
    _lib.check(lib.syn_fb_create(0, C.byref(fresh)))
    assert lib.syn_fb_forward_batch(fresh, stack.data_ptr(), 2, h, w, loc.data_ptr(), conf.data_ptr(), None) == 3       # not committed
    lib.syn_fb_destroy(fresh)
    torch.cuda.synchronize()
    assert net.launch_count - n0 <= 6                                              # only the wrong-size debug stop got as far as launching
    again = net.forward_batch(stack)
    torch.cuda.synchronize()
    assert torch.equal(again[0], good[0]) and torch.equal(again[1], good[1])
    assert fb.detect_batch(frames) == [fb(frames[0]), fb(frames[1])]


def test_workspace_growth_keeps_results(sd):
    """One handle: a one-image call, a larger stack (the workspace grows), a smaller one, another size, the first again."""
    net = faceboxes.FaceBoxesNet(sd, DEV)
    a = torch.from_numpy(_frames(6, 120, 96)).to(DEV)
    b = torch.from_numpy(_frames(2, 250, 333)).to(DEV)
    one = net.forward(a[0])
    six = net.forward_batch(a)
    two = net.forward_batch(a[:2].contiguous())
    other = net.forward_batch(b)
    back = net.forward_batch(a)
    torch.cuda.synchronize()
    assert torch.equal(six[0][0], one[0]) and torch.equal(six[1][0], one[1])
    assert torch.equal(two[0], six[0][:2]) and torch.equal(back[0], six[0]) and torch.equal(back[1], six[1])
    assert torch.equal(other[0][1], net.forward(b[1])[0])
    net.close()
