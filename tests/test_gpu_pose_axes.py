"""The pose axes on the H100: syn_draw_lines against the host emulation of the same header (which
test_draw_emulation.py holds to cv2.line), draw_axis against the reference's own draw_axis (the committed golden digests),
and the models' pose_overlay_batch / pose_overlay_images against the per-frame loop of get_all_outputs + draw_axis they
replace.  Every equality is byte for byte."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from golden.make_golden_axis import base_image
from golden.make_golden_draw import digest
from oracle import synth_mbv1, synth_model, synth_resnet
from oracle.stage_check import make_model
from synergynet_b200 import _lib, faceboxes, synthetic
from synergynet_b200.inference import ImagePack, _segment_table, draw_axis, draw_lines_device, pack_images

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def emul():
    out = os.path.join(tempfile.mkdtemp(prefix='draw_emul_'), 'libdraw_emul.so')
    subprocess.run(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', out, os.path.join(HERE, 'host_emul', 'draw_emul.cpp')],
                   check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.emul_draw_lines.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int]
    return lib


def emul_draw(lib, img, segs):
    out = np.ascontiguousarray(img).copy()
    a = np.array([[x0, y0, x1, y1, b | (g << 8) | (r << 16)] for x0, y0, x1, y1, (b, g, r) in segs], np.int64).reshape(-1, 5)
    a = np.ascontiguousarray(a.astype(np.int32))
    lib.emul_draw_lines(out.ctypes.data, out.shape[0], out.shape[1], a.ctypes.data, a.shape[0])
    return out


def _segments(rng, h, w, n):
    """n segments crowding a few centres (heavy overlap, so the draw order decides bytes), some leaving the image, some
    far outside, some of length 0."""
    centres = rng.uniform(-0.1, 1.1, (3, 2)) * (w, h)
    out = []
    for k in range(n):
        c = centres[k % 3]
        if k % 11 == 10:
            p0 = [int(v) for v in rng.integers(-(1 << 30), 1 << 30, 2)]
        else:
            p0 = [int(c[0] + rng.normal(0, 6)), int(c[1] + rng.normal(0, 6))]
        r = 0 if k % 7 == 6 else rng.uniform(1, max(2.0, 0.6 * max(h, w)))
        a = rng.uniform(0, 2 * np.pi)
        p1 = [int(p0[0] + r * np.cos(a)), int(p0[1] + r * np.sin(a))]
        out.append((*p0, *p1, tuple(int(v) for v in rng.integers(0, 256, 3))))
    return out


@pytest.mark.parametrize('n', [1, 4, 16, 64])
def test_kernel_equals_emulation_on_frame_stacks(emul, n):
    rng = np.random.default_rng(n)
    frames = np.stack([synthetic.make_scene_u8(720, 1080, 3 * i + n) for i in range(n)])
    segs = [[] if i == 1 else _segments(rng, 720, 1080, int(rng.integers(1, 49))) for i in range(n)]
    stack = torch.from_numpy(frames).to(DEV)
    out = draw_lines_device(stack, segs)
    assert out is stack
    got = stack.cpu().numpy()
    for i in range(n):
        assert np.array_equal(got[i], emul_draw(emul, frames[i], segs[i])), f'frame {i} ({len(segs[i])} segments)'
    if n > 1:
        assert np.array_equal(got[1], frames[1])


def test_kernel_equals_emulation_on_image_packs(emul):
    """Mixed sizes, segments leaving every image: the neighbours' bytes are those of their own segments only."""
    rng = np.random.default_rng(5)
    sizes = [(360, 480), (1, 1), (250, 333), (720, 1080), (97, 61), (1, 40), (40, 1), (5, 7)]
    images = [synthetic.make_scene_u8(h, w, 11 * i) for i, (h, w) in enumerate(sizes)]
    segs = [_segments(rng, h, w, 20) for h, w in sizes]
    segs[4] = []
    pack = pack_images(images, DEV)
    draw_lines_device(pack, segs)
    for i, im in enumerate(images):
        got = pack.image(i).cpu().numpy()
        assert np.array_equal(got, emul_draw(emul, im, segs[i])), f'image {i} {sizes[i]}'
    assert np.array_equal(pack.image(4).cpu().numpy(), images[4])


def _axis_cases():
    doc = json.load(open(os.path.join(HERE, 'golden', 'axis_golden.json')))
    z = np.load(os.path.join(HERE, 'golden', 'axis_golden.npz'))
    for i, case in enumerate(doc['cases']):
        h, w = (int(v) for v in z[f'hw{i}'])
        faces = [(*[float(a) for a in z[f'ang{i}'][k]], z[f'pts{i}'][k]) for k in range(len(z[f'ang{i}']))]
        yield i, base_image(i, h, w), faces, case


@pytest.mark.parametrize('on_device', [False, True])
def test_draw_axis_equals_the_reference(on_device):
    kinds = {'ValueError': ValueError, 'OverflowError': OverflowError, 'error': OverflowError}
    for i, img, faces, case in _axis_cases():
        canvas = torch.from_numpy(img.copy()).to(DEV) if on_device else img.copy()
        err = None
        try:
            with np.errstate(all='ignore'):
                for yaw, pitch, roll, pts in faces:
                    assert draw_axis(canvas, yaw, pitch, roll, 0.0, 0.0, size=50, pts68=pts) is canvas
        except (ValueError, OverflowError) as e:
            err = e
        got = canvas.cpu().numpy() if on_device else canvas
        assert digest(got) == case['digest'], i
        if case['error'] is None:
            assert err is None, (i, err)
        else:
            assert type(err) is kinds[case['error']], (i, err)


def test_draw_entry_replays_in_a_cuda_graph(emul):
    """Captured after an eager call, replayed on new segments (same counts, rewritten in the captured buffer): every
    replay equals an eager call."""
    lib = _lib.load()
    rng = np.random.default_rng(9)
    n, h, w = 4, 200, 300
    frames = torch.from_numpy(np.stack([synthetic.make_scene_u8(h, w, i) for i in range(n)])).to(DEV)
    counts = [5, 0, 12, 3]
    table_host = np.array([[3 * h * w * i, h, w] for i in range(n)], np.int64)

    def seg_lists():
        return [_segments(rng, h, w, c) for c in counts]

    segs0 = seg_lists()
    buf, (a, b), n_segs, start = _segment_table(segs0, table_host)
    table = torch.from_numpy(buf).to(DEV)
    canvas = frames.clone()

    def call():
        _lib.check(lib.syn_draw_lines(canvas.data_ptr(), canvas.numel(), table_host.ctypes.data, table.data_ptr(), n, start.ctypes.data,
                                      table[a:b].data_ptr(), table[b:].data_ptr(), n_segs, 4, 8,
                                      torch.cuda.current_stream(DEV).cuda_stream))

    call()                                                          # eager first
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    for rep in range(3):
        segs = seg_lists()
        table.copy_(torch.from_numpy(_segment_table(segs, table_host)[0]).to(DEV))
        canvas.copy_(frames)
        g.replay()
        torch.cuda.synchronize()
        replayed = canvas.cpu().numpy()
        eager = frames.clone()
        draw_lines_device(eager, segs)
        assert np.array_equal(replayed, eager.cpu().numpy()), rep
        for i in range(n):
            assert np.array_equal(replayed[i], emul_draw(emul, frames[i].cpu().numpy(), segs[i])), (rep, i)


# ---- the models -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def synth_pack():
    from synergynet_b200.params import ParamsPack, set_param_pack
    set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))


@pytest.fixture(scope='module')
def fb():
    return faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0), device='cuda:0')


def _checkpoint(arch):
    if arch == 'mobilenet_v2':
        return make_model(synth_model.build_state_dict(0))
    if arch.startswith('resnet'):
        return make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
    return make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)


def _loop(img, outputs):
    """singleImage.py:112-117 on one frame: draw_axis per face onto a copy, fed with get_all_outputs' results."""
    canvas = img.copy()
    lmks, _, poses = outputs
    for (angles, translation), lmk in zip(poses, lmks):
        canvas = draw_axis(canvas, angles[0], angles[1], angles[2], translation[0], translation[1], size=50, pts68=lmk)
    return canvas


RECTS = [[[100.0, 80.0, 300.0, 300.0, 0.9], [250.0, 150.0, 420.0, 330.0, 0.8], [-40.0, 500.0, 120.0, 700.0, 0.7]], [],
         [[600.0, 200.0, 900.0, 520.0, 0.9]], [[1.0, 1.0, 60.0, 80.0, 0.6], [900.0, 600.0, 1100.0, 760.0, 0.9]]]


@pytest.mark.parametrize('arch', ['mobilenet_v2', 'resnet18', 'mobilenet_05'])
def test_pose_overlay_batch_equals_the_per_frame_loop(synth_pack, fb, arch):
    model = _checkpoint(arch)
    frames = np.stack([synthetic.make_scene_u8(720, 1080, 50 + i) for i in range(4)])
    outputs = model.get_all_outputs_batch(frames, rects=RECTS)
    want = [_loop(frames[i], outputs[i]) for i in range(4)]
    got = model.pose_overlay_batch(frames, rects=RECTS)
    assert isinstance(got, np.ndarray) and got.shape == frames.shape
    for i in range(4):
        assert np.array_equal(got[i], want[i]), f'{arch} frame {i}'
    assert np.array_equal(got[1], frames[1]) and (got[0] != frames[0]).any()
    on_dev = model.pose_overlay_batch(torch.from_numpy(frames).to(DEV), rects=RECTS)
    assert isinstance(on_dev, torch.Tensor) and on_dev.is_cuda and np.array_equal(on_dev.cpu().numpy(), got)
    model.face_detector = fb
    try:
        small = np.stack([synthetic.make_scene_u8(480, 640, 80 + i) for i in range(3)])
        auto = model.pose_overlay_batch(small)
        outs = model.get_all_outputs_batch(small)
        for i in range(3):
            assert np.array_equal(auto[i], _loop(small[i], outs[i])), f'{arch} detected frame {i}'
    finally:
        model.face_detector = None


@pytest.mark.parametrize('arch', ['mobilenet_v2', 'resnet18'])
def test_pose_overlay_images_equals_the_per_image_loop(synth_pack, fb, arch):
    model = _checkpoint(arch)
    sizes = [(360, 480), (1, 1), (250, 333), (720, 1080)]
    images = [synthetic.make_scene_u8(h, w, 7 * i) for i, (h, w) in enumerate(sizes)]
    rects = [[[10.0, 20.0, 200.0, 240.0, 0.9], [150.0, 100.0, 330.0, 300.0, 0.8]], [], [[-30.0, 40.0, 120.0, 200.0, 0.7]],
             [[500.0, 300.0, 800.0, 620.0, 0.9]]]
    outputs = model.get_all_outputs_images(images, rects=rects)
    got = model.pose_overlay_images(images, rects=rects)
    assert isinstance(got, list) and len(got) == 4
    for i in range(4):
        assert np.array_equal(got[i], _loop(images[i], outputs[i])), f'{arch} image {i}'
    assert np.array_equal(got[1], images[1])
    dev = model.pose_overlay_images([torch.from_numpy(im).to(DEV) for im in images], rects=rects)
    assert all(isinstance(t, torch.Tensor) and t.is_cuda for t in dev)
    assert all(np.array_equal(dev[i].cpu().numpy(), got[i]) for i in range(4))
    model.face_detector = fb
    try:
        small = [synthetic.make_scene_u8(h, w, 3 + h) for h, w in ((240, 320), (300, 200))]
        auto = model.pose_overlay_images(small)
        outs = model.get_all_outputs_images(small)
        for i in range(2):
            assert np.array_equal(auto[i], _loop(small[i], outs[i])), f'{arch} detected image {i}'
    finally:
        model.face_detector = None


def test_pose_overlay_leaves_the_other_outputs_unchanged(synth_pack):
    model = _checkpoint('mobilenet_v2')
    frames = np.stack([synthetic.make_scene_u8(720, 1080, 90 + i) for i in range(4)])
    before_o = model.overlay_batch(frames, rects=RECTS)
    before_g = model.get_all_outputs_batch(frames, rects=RECTS)
    model.pose_overlay_batch(frames, rects=RECTS)
    after_o = model.overlay_batch(frames, rects=RECTS)
    after_g = model.get_all_outputs_batch(frames, rects=RECTS)
    assert all(np.array_equal(a, b) for a, b in zip(before_o, after_o))
    for (l0, m0, p0), (l1, m1, p1) in zip(before_g, after_g):
        assert all(np.array_equal(a, b) for a, b in zip(l0, l1)) and all(np.array_equal(a, b) for a, b in zip(m0, m1))
        assert all(a[0] == b[0] and np.array_equal(a[1], b[1]) for a, b in zip(p0, p1))


def test_pose_overlay_names_the_failing_face(synth_pack):
    model = _checkpoint('mobilenet_v2')
    frames = np.stack([synthetic.make_scene_u8(240, 320, 1 + i) for i in range(2)])
    import synergynet_b200.model_building as mb
    real = mb.plan_axis

    def failing(yaw, pitch, roll, pts68):
        return [], ValueError('cannot convert float NaN to integer')

    mb.plan_axis = failing
    try:
        with pytest.raises(ValueError, match=r'frame 1, face 0: cannot convert float NaN'):
            model.pose_overlay_batch(frames, rects=[[], [[10.0, 10.0, 100.0, 120.0, 0.9]]])
    finally:
        mb.plan_axis = real
