"""CPU checks of the crop + resize kernel's arithmetic without a GPU: tests/host_emul/resize_emul.cpp compiles
csrc/resize_math.h -- the header the CUDA kernel is built from -- with g++ and runs its per-pixel function as serial loops
over the plan the library's host planner builds.  The bytes must be live cv2.resize's (after crop_img for face ROIs).
Also covers the planner's and the device entry's argument checks, which run before any CUDA work."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from golden import make_golden_resize as gr
from synergynet_b200 import _lib, synthetic
from synergynet_b200.inference import INTER_LANCZOS4, INTER_LINEAR, crop_img, roi_ints, resize_plan

cv2 = pytest.importorskip('cv2')

HERE = os.path.dirname(os.path.abspath(__file__))
MODES = (INTER_LINEAR, INTER_LANCZOS4)
V, I, L = C.c_void_p, C.c_int, C.c_longlong


@pytest.fixture(scope='module')
def emul():
    out = os.path.join(tempfile.mkdtemp(prefix='resize_emul_'), 'libresize_emul.so')
    subprocess.run(['g++', '-O2', '-shared', '-fPIC', '-o', out, os.path.join(HERE, 'host_emul', 'resize_emul.cpp')],
                   check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.emul_crop_resize.argtypes = [V, I, I, V, I, I, I, I, V, L, L, L, L]
    lib.emul_lanczos4_tap_sums.argtypes = [C.c_float, V, V]
    return lib


def emul_crop_resize(emul, img, boxes, out_h, out_w, mode, planar=False):
    """The kernel's result for every box on the CPU: (B,h,w,3), or (B,3,h,w) when ``planar``."""
    img = np.ascontiguousarray(img)
    rois = np.array([roi_ints(b) for b in boxes], np.int32)
    plan = resize_plan(rois, out_h, out_w, mode)
    B = len(boxes)
    if planar:
        out = np.zeros((B, 3, out_h, out_w), np.uint8)
        strides = (3 * out_h * out_w, out_w, 1, out_h * out_w)
    else:
        out = np.zeros((B, out_h, out_w, 3), np.uint8)
        strides = (3 * out_h * out_w, 3 * out_w, 3, 1)
    emul.emul_crop_resize(img.ctypes.data, img.shape[0], img.shape[1], plan.ctypes.data, B, out_h, out_w, mode, out.ctypes.data, *strides)
    return out


def images(h, w, seed):
    rng = np.random.default_rng(seed)
    checker = ((np.add.outer(np.arange(h), np.arange(w)) % 2) * 255).astype(np.uint8)
    return {'random': rng.integers(0, 256, (h, w, 3), dtype=np.uint8),
            'const255': np.full((h, w, 3), 255, np.uint8),
            'checker': np.repeat(checker[:, :, None], 3, axis=2)}


SIDES = list(range(1, 521)) + [119, 120, 121, 239, 240, 241, 480]


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('content', ['random', 'const255', 'checker'])
def test_sides_to_120_match_cv2(emul, mode, content):
    """Every source side 1..520 (plus the ones around 120 and the exact halving), square and non-square, cut as a batch of
    ROIs from one image and resized to 120 x 120."""
    img = images(530, 530, 11)[content]
    boxes = []
    for s in SIDES:
        other = (s * 7) % 520 + 1
        boxes.append([s % 9, s % 5, s % 9 + s, s % 5 + s])
        boxes.append([3, 1, 3 + other, 1 + s])
    got = emul_crop_resize(emul, img, boxes, 120, 120, mode)
    for b, box in enumerate(boxes):
        want = cv2.resize(crop_img(img, box), dsize=(120, 120), interpolation=mode)
        assert np.array_equal(got[b], want), (box, mode, content)


@pytest.mark.parametrize('content', ['random', 'checker'])
def test_detector_shrinks_match_cv2(emul, content):
    """FaceBoxes.__call__'s shrink of images above 720 x 1080 (cv2.resize's default INTER_LINEAR), including the exact
    halving of 1440 x 2160 that OpenCV turns into its 2 x 2 area path."""
    for k, (h, w) in enumerate(gr.SHRINKS):
        img = images(h, w, k)[content]
        hs, ws = gr.detector_size(h, w)
        got = emul_crop_resize(emul, img, [[0, 0, w, h]], hs, ws, INTER_LINEAR)[0]
        assert np.array_equal(got, cv2.resize(img, dsize=(ws, hs))), (h, w)


@pytest.mark.parametrize('mode', MODES)
def test_rois_outside_the_image_and_planar_layout(emul, mode):
    """ROIs partly and wholly outside the image (crop pixels there are 0; the resampler replicates that fill at the crop's
    border), fractional boxes rounded half-even, written in the backbone's planar (B,3,120,120) layout."""
    scene = synthetic.make_scene_u8(*gr.SCENE)
    got = emul_crop_resize(emul, scene, gr.ROIS, 120, 120, mode, planar=True)
    for b, box in enumerate(gr.ROIS):
        want = cv2.resize(gr.host_crop(scene, box), dsize=(120, 120), interpolation=mode)
        assert np.array_equal(got[b].transpose(1, 2, 0), want), (box, mode)


def test_host_crop_is_crop_img_where_the_box_meets_the_image():
    scene = synthetic.make_scene_u8(*gr.SCENE)
    met = 0
    for box in gr.ROIS:
        x0, y0, x1, y1 = roi_ints(box)
        if min(x1, scene.shape[1]) > max(x0, 0) and min(y1, scene.shape[0]) > max(y0, 0):
            assert np.array_equal(gr.host_crop(scene, box), crop_img(scene, box))
            met += 1
        else:
            assert not gr.host_crop(scene, box).any()
    assert met == len(gr.ROIS) - 3


def test_committed_cv2_digests(emul):
    """The emulation reproduces the crops and shrinks recorded from cv2 in tests/golden/resize_digests.json."""
    with open(os.path.join(HERE, 'golden', 'resize_digests.json')) as f:
        gold = json.load(f)
    scene = synthetic.make_scene_u8(*gr.SCENE)
    for name, mode in gr.MODES.items():
        got = emul_crop_resize(emul, scene, gr.ROIS, 120, 120, mode)
        assert [gr.digest(c) for c in got] == gold['crops'][name], name
    for k, (h, w) in enumerate(gr.SHRINKS[:2]):                      # the large ones are covered against live cv2 above
        hs, ws = gr.detector_size(h, w)
        got = emul_crop_resize(emul, synthetic.make_scene_u8(h, w, k), [[0, 0, w, h]], hs, ws, INTER_LINEAR)[0]
        assert gr.digest(got) == gold['shrinks'][f'{h}x{w}']


def test_lanczos4_sums_stay_in_int32(emul):
    """resize_math.h's int32 bound: the positive / negative fixed-point Lanczos4 taps sum to at most 2780 / 732."""
    pos, neg = C.c_int(), C.c_int()
    P = N = 0
    for f in np.linspace(0, 1, 200_001, endpoint=False, dtype=np.float32):
        emul.emul_lanczos4_tap_sums(C.c_float(float(f)), C.byref(pos), C.byref(neg))
        P, N = max(P, pos.value), max(N, neg.value)
    assert P <= 2780 and N <= 732, (P, N)
    assert 255 * (P * P + N * N) + (1 << 21) < 2 ** 31 - 1


def test_planner_and_entry_reject_bad_arguments():
    lib = _lib.load()
    ok = np.array([[0, 0, 10, 10]], np.int32)
    n = lib.syn_crop_resize_plan_size(1, 120, 120, INTER_LANCZOS4)
    assert n == 32 + 240 * (4 + 16) and lib.syn_crop_resize_plan_size(1, 120, 120, INTER_LINEAR) == 32 + 240 * (4 + 4)
    assert lib.syn_crop_resize_plan_size(1, 120, 120, 2) == -1 and lib.syn_crop_resize_plan_size(0, 120, 120, 1) == -1
    plan = np.zeros(n, np.uint8)

    def planner(rois, out_h=120, out_w=120, mode=INTER_LANCZOS4, nbytes=n):
        rois = np.asarray(rois, np.int32)
        return lib.syn_crop_resize_plan_host(rois.ctypes.data, rois.shape[0], out_h, out_w, mode, plan.ctypes.data, nbytes)
    assert planner(ok) == 0
    for empty in ([[5, 0, 5, 10]], [[0, 7, 10, 7]], [[9, 0, 3, 10]]):         # cv2.resize raises on an empty crop
        assert planner(empty) == 4 and b'empty' in lib.syn_last_error()
    assert planner(ok, out_h=0) == 1 and planner(ok, out_w=-3) == 1
    assert planner(ok, mode=3) == 6 and planner(ok, mode=0) == 6           # INTER_AREA / INTER_NEAREST are not built
    assert planner(ok, nbytes=n - 1) == 4
    with pytest.raises(_lib.SynergyLibError, match='SYN_ERR_SHAPE'):
        resize_plan(np.array([[0, 0, 0, 4]], np.int32), 120, 120, INTER_LINEAR)
    one = C.c_void_p(8)     # never dereferenced: the calls below fail validation before any CUDA work
    args = lambda ch=3, mode=INTER_LINEAR, oh=120, img=one: (img, 64, 64, ch, one, 1, oh, 120, mode, one, 43200, 120, 1, 14400, None)
    assert lib.syn_crop_resize(*args(ch=1)) == 6 and lib.syn_crop_resize(*args(ch=4)) == 6
    assert lib.syn_crop_resize(*args(mode=2)) == 6
    assert lib.syn_crop_resize(*args(oh=0)) == 1 and lib.syn_crop_resize(*args(img=None)) == 1


def test_crop_resize_device_needs_a_cuda_image():
    import torch
    from synergynet_b200.inference import crop_resize_device
    with pytest.raises(ValueError, match='CUDA'):
        crop_resize_device(torch.zeros((8, 8, 3), dtype=torch.uint8), [[0, 0, 4, 4]])
