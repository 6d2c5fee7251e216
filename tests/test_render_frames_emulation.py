"""CPU checks of the frame-axis render stage without a GPU: tests/host_emul/render_frames_emul.cpp compiles
csrc/render_math.h -- the header the CUDA kernels are built from -- with g++.  The overlay blend must give OpenCV's
``cv2.addWeighted`` bytes for every uint8 pair, live and against the committed digests; the per-mesh pixel boxes must hold
every pixel the depth pass keys.  Also the argument checks of the new C entries, which fail before any CUDA work."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from golden.make_golden_add_weighted import cv2_body, cv2_tail
from synergynet_b200 import _lib, synthetic

HERE = os.path.dirname(os.path.abspath(__file__))
DIGESTS = os.path.join(HERE, 'golden', 'add_weighted_digests.json')
ALPHAS = (0.0, 0.1, 0.3, 0.5, 0.6, 0.75, 1.0)


def P(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope='module')
def emul():
    out = os.path.join(tempfile.mkdtemp(prefix='render_frames_emul_'), 'librender_frames_emul.so')
    subprocess.run(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', out,
                    os.path.join(HERE, 'host_emul', 'render_frames_emul.cpp')], check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.emul_add_weighted.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_double]
    lib.emul_frame_plan.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                    C.c_int, C.c_void_p, C.c_void_p]
    lib.emul_frame_keys.argtypes = lib.emul_frame_plan.argtypes[:10] + [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.emul_frame_keys.restype = C.c_longlong
    return lib


def _pairs():
    i = np.arange(65536)
    return (i // 256).astype(np.uint8), (i % 256).astype(np.uint8)


def _emul_blend(emul, a, b, alpha):
    out = np.empty_like(a)
    emul.emul_add_weighted(P(a), P(b), P(out), a.size, float(alpha))
    return out


def _digest(x):
    return hashlib.sha256(np.ascontiguousarray(x, np.uint8).tobytes()).hexdigest()


def _unfused(a, b, alpha):
    """a * (1 - alpha) + b * alpha in float32 with two roundings before the add, then cv2's rounding and clamp."""
    wa, wb = np.float32(1 - alpha), np.float32(alpha)
    v = a.astype(np.float32) * wa + b.astype(np.float32) * wb
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)


@pytest.mark.parametrize('alpha', ALPHAS)
def test_add_weighted_equals_live_cv2_for_every_pair(emul, alpha):
    """Body position (one long continuous row: OpenCV's SIMD loop) and tail position (rows of three elements: its scalar
    loop), all 65 536 (a, b) pairs."""
    cv2 = pytest.importorskip('cv2')
    a, b = _pairs()
    got = _emul_blend(emul, a, b, alpha)
    assert np.array_equal(got, cv2_body(a, b, alpha))
    assert np.array_equal(got, cv2_tail(a, b, alpha))
    for k in (0, 1, 255, 256 * 77 + 13, 65535):                       # and as the reference calls it, on 3-element images
        ia, ib = np.full((1, 1, 3), a[k], np.uint8), np.full((1, 1, 3), b[k], np.uint8)
        assert (cv2.addWeighted(ia, 1 - alpha, ib, alpha, 0) == got[k]).all()


@pytest.mark.parametrize('alpha', [-0.5, 0.05, 0.123456789, 1.7, 37.25, -1e3, 1e9, -1e9])
def test_add_weighted_saturates_as_cv2_for_any_finite_alpha(emul, alpha):
    cv2 = pytest.importorskip('cv2')
    a, b = _pairs()
    got = _emul_blend(emul, a, b, alpha)
    assert np.array_equal(got, cv2.addWeighted(a.reshape(1, -1), 1 - alpha, b.reshape(1, -1), alpha, 0).reshape(-1))


def test_add_weighted_matches_the_committed_digests(emul):
    doc = json.load(open(DIGESTS))
    assert doc['alphas'] == list(ALPHAS)
    a, b = _pairs()
    for alpha in ALPHAS:
        d = _digest(_emul_blend(emul, a, b, alpha))
        assert d == doc['body'][repr(alpha)] == doc['tail'][repr(alpha)], alpha


def test_unfused_blend_fails_the_digest():
    """The digests tell the fused form from a * (1 - alpha) + b * alpha: at alpha = 0.1 the unfused bytes differ (733 pairs),
    at 0.6 (the reference's alpha) they happen to agree."""
    doc = json.load(open(DIGESTS))
    a, b = _pairs()
    assert _digest(_unfused(a, b, 0.1)) != doc['body']['0.1']
    assert _digest(_unfused(a, b, 0.6)) == doc['body']['0.6']


def test_unfused_blend_differs_from_cv2_where_the_fma_matters(emul):
    a, b = _pairs()
    got, unf = _emul_blend(emul, a, b, 0.1), _unfused(a, b, 0.1)
    assert int((got != unf).sum()) == 733


# ---- the per-mesh pixel boxes ----------------------------------------------------------------------------------------------------
def _meshes(seed, h, w):
    """Seeded (M,3,nver) plane-major meshes: on the canvas, partly off every edge, wholly off, and with degenerate and
    out-of-range triangles in the topology."""
    rows, cols = 9, 11
    tri = synthetic.make_render_topology(rows, cols)
    nver = rows * cols
    v = synthetic.make_render_meshes(6, h, w, seed=seed, rows=rows, cols=cols, size=min(h, w) / 2.5)
    v[1, 0] -= 0.6 * w                                                  # partly off the left edge
    v[2, 1] += 0.6 * h                                                  # partly off the bottom
    v[3, 0] += 3.0 * w                                                  # wholly off the canvas
    v[4, :2] *= 0.25                                                    # a small mesh near the origin
    v[5, :2, : nver // 2] = v[5, :2, :1]                               # half its vertices collapsed onto one point
    bad = np.array([[0, 0, 0], [1, 1, 2], [3, nver + 5, 4], [-1, 2, 3]], np.int32)    # degenerate and out-of-range triangles
    tri = np.ascontiguousarray(np.concatenate([tri, bad]))
    return np.ascontiguousarray(v), tri, nver


def _box_of(v, tri, nver, h, w):
    """The union of the clamped triangle boxes, in numpy (float32 floor / ceil like tri_setup)."""
    ok = ((tri >= 0) & (tri < nver)).all(1)
    t = tri[ok]
    x, y = v[0][t], v[1][t]
    x0 = np.maximum(np.floor(x.min(1)).astype(np.int64), 0)
    x1 = np.minimum(np.ceil(x.max(1)).astype(np.int64), w - 1)
    y0 = np.maximum(np.floor(y.min(1)).astype(np.int64), 0)
    y1 = np.minimum(np.ceil(y.max(1)).astype(np.int64), h - 1)
    live = (x1 >= x0) & (y1 >= y0)
    if not live.any():
        return [0, 0, -1, -1]
    return [int(x0[live].min()), int(y0[live].min()), int(x1[live].max()), int(y1[live].max())]


@pytest.mark.parametrize('seed,h,w', [(0, 48, 64), (1, 37, 91), (2, 80, 45), (3, 1, 70), (4, 64, 1)])
def test_mesh_boxes_hold_every_keyed_pixel(emul, seed, h, w):
    v, tri, nver = _meshes(seed, h, w)
    m = v.shape[0]
    boxes = np.zeros((m, 4), np.int32)
    off = np.zeros(m + 1, np.int64)
    args = (P(v), 3 * nver, 1, nver, m, nver, P(tri), tri.shape[0], h, w)
    emul.emul_frame_plan(*args, P(boxes), P(off))
    areas = [(b[2] - b[0] + 1) * (b[3] - b[1] + 1) if b[2] >= b[0] else 0 for b in boxes]
    assert off.tolist() == np.concatenate([[0], np.cumsum(areas)]).tolist()
    for b in range(m):
        assert boxes[b].tolist() == _box_of(v[b], tri, nver, h, w), b
    assert areas[3] == 0 and boxes[3].tolist() == [0, 0, -1, -1]         # wholly off the canvas: no key slot
    keys = np.zeros(max(int(off[-1]), 1), np.uint64)
    full = np.zeros((m, h, w), np.uint64)
    assert emul.emul_frame_keys(*args, P(boxes), P(off), P(keys), P(full)) == 0
    # the box keys are the full-canvas keys: every keyed pixel sits in its box, every box slot is that pixel's key
    for b in range(m):
        x0, y0, x1, y1 = boxes[b]
        inside = full[b, y0:y1 + 1, x0:x1 + 1] if x1 >= x0 else full[b, :0, :0]
        assert full[b].astype(bool).sum() == inside.astype(bool).sum()
        assert np.array_equal(keys[off[b]:off[b + 1]], inside.reshape(-1))
    assert full.any() and int(off[-1]) < m * h * w


# ---- C entries: argument checks before any CUDA work ----------------------------------------------------------------------------
def _fails(code, want, text):
    assert code == want, (code, _lib.load().syn_last_error())
    assert text in _lib.load().syn_last_error(), _lib.load().syn_last_error()


def test_frame_entries_reject_bad_arguments():
    lib = _lib.load()
    p = C.c_void_p(8)                                      # never dereferenced: every call below fails validation first
    start = np.array([0, 2, 2, 5], np.int32)
    ms = start.ctypes.data

    def plan(v=p, m=5, nver=10, tri=p, ntri=4, st=ms, nf=3, h=16, w=16, boxes=p, off=p, sv=1, sc=10):
        return lib.syn_render_frames_plan(v, 30, sv, sc, m, nver, tri, ntri, st, nf, h, w, boxes, off, None)

    _fails(plan(v=None), 1, b'syn_render_frames_plan: null pointer')
    _fails(plan(st=None), 1, b'null pointer')
    _fails(plan(m=0), 1, b'no mesh')
    _fails(plan(sv=0), 1, b'non-positive stride')
    _fails(plan(nf=0), 1, b'0 frames')
    _fails(plan(m=70000, st=np.array([0, 70000], np.int32).ctypes.data, nf=1), 1, b'1..65535')
    _fails(plan(h=0), 1, b'frame size 0x16')
    _fails(plan(tri=None), 1, b'null pointer or negative triangle count')
    _fails(plan(boxes=None), 1, b'null pointer')
    for bad, text in (([1, 2, 2, 5], b'must run from 0 to 5'), ([0, 2, 2, 4], b'must run from 0 to 5'),
                      ([0, 3, 2, 5], b'not monotone at frame 1 (2 after 3)')):
        arr = np.array(bad, np.int32)
        _fails(plan(st=arr.ctypes.data), 4, text)

    def rast(fr=p, sol=p, nf=3, c=3, cc=3, st=ms, std=p, nkeys=100, ws=100, keys=p, m=5, off=p):
        return lib.syn_rasterize_frames(fr, sol, nf, 16, 16, c, p, 30, 1, 10, m, 10, p, 4, p, cc, st, std, p, off, nkeys, keys, ws, None)

    _fails(rast(fr=None), 1, b'syn_rasterize_frames: null pointer')
    _fails(rast(sol=None), 1, b'null pointer')
    _fails(rast(std=None), 1, b'null pointer')
    _fails(rast(keys=None), 1, b'null pointer')
    _fails(rast(off=None), 1, b'null pointer')
    _fails(rast(cc=4), 4, b'3 image channels, colours of 4 channels')
    _fails(rast(c=0, cc=0), 4, b'0 image channels')
    _fails(rast(ws=99), 4, b'key workspace of 99 slots, the plan needs 100')
    _fails(rast(nkeys=-1), 4, b'key workspace')
    _fails(rast(st=np.array([0, 4, 2, 5], np.int32).ctypes.data), 4, b'not monotone at frame 1')
    _fails(rast(nf=65536), 1, b'65536 frames')
    _fails(lib.syn_add_weighted_u8(None, p, 0.6, p, 10, None), 1, b'syn_add_weighted_u8: null pointer')
    _fails(lib.syn_add_weighted_u8(p, p, 0.6, None, 10, None), 1, b'null pointer')
    _fails(lib.syn_add_weighted_u8(p, p, 0.6, p, -1, None), 1, b'negative size')
    for alpha in (float('nan'), float('inf'), -float('inf')):
        _fails(lib.syn_add_weighted_u8(p, p, alpha, p, 10, None), 1, b'is not finite')
    assert lib.syn_add_weighted_u8(p, p, 0.6, p, 0, None) == 0             # nothing to do: no launch


def test_render_batch_refuses_mismatched_lists():
    from synergynet_b200 import Sim3DR
    frames = np.zeros((2, 4, 5, 3), np.uint8)
    with pytest.raises(ValueError, match='1 mesh lists'):
        Sim3DR.render_batch(frames, [[]], np.zeros((1, 3), np.int32))
    with pytest.raises(ValueError, match='3 paths for 2 frames'):
        Sim3DR.render_batch(frames, [[], []], np.zeros((1, 3), np.int32), wfps=['a.png', None, None])
