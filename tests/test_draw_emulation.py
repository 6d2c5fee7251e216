"""CPU checks of the pose-axis drawing without a GPU: tests/host_emul/draw_emul.cpp compiles csrc/draw_math.h -- the
header the CUDA kernel is built from -- with g++.  It must give OpenCV's cv2.line(img, p0, p1, colour, 4) bytes, live
and against the committed digests, while variants that change one rounding step must not; the host end-point planner
plus the emulation must reproduce what the reference's own draw_axis drew and raised (tests/golden/axis_golden.*).
Also the argument checks of syn_draw_lines, which fail before any CUDA work."""
import ctypes as C
import json
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

from golden.make_golden_axis import base_image, ends64
from golden.make_golden_draw import DIGEST_SETS, SIZES, cv2_draw, digest, draw_cases
from synergynet_b200 import _lib
from synergynet_b200.inference import AXIS_COLOURS, plan_axis

HERE = os.path.dirname(os.path.abspath(__file__))
DIGESTS = os.path.join(HERE, 'golden', 'draw_digests.json')
AXIS_NPZ = os.path.join(HERE, 'golden', 'axis_golden.npz')
AXIS_JSON = os.path.join(HERE, 'golden', 'axis_golden.json')


def P(a):
    return a.ctypes.data_as(C.c_void_p)


def _build(variant=0):
    out = os.path.join(tempfile.mkdtemp(prefix='draw_emul_'), f'libdraw_emul{variant}.so')
    subprocess.run(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', f'-DSYN_DRAW_VARIANT={variant}', '-o', out,
                    os.path.join(HERE, 'host_emul', 'draw_emul.cpp')], check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.emul_draw_lines.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int]
    return lib


@pytest.fixture(scope='module')
def emul():
    return _build()


def emul_draw(lib, img, segs):
    out = np.ascontiguousarray(img).copy()
    segs = np.ascontiguousarray(segs, np.int32).reshape(-1, 5)
    lib.emul_draw_lines(P(out), out.shape[0], out.shape[1], P(segs), segs.shape[0])
    return out


@pytest.mark.parametrize('seed', range(4))
def test_emulation_equals_live_cv2(emul, seed):
    """4 x 25 000 segments: every octant, lengths 0, 1 and long, ends on, just inside and just outside each border, far
    outside (up to +-2^30 and the int32 edges), canvases 1x1, 1xW, Hx1 and odd sizes, overlapping sequences of colours."""
    pytest.importorskip('cv2')
    n = 0
    for img, segs in draw_cases(100 + seed, 2700, 19):
        n += len(segs)
        got, want = emul_draw(emul, img, segs), cv2_draw(img, segs)
        assert np.array_equal(got, want), (img.shape, segs.tolist(), np.argwhere((got != want).any(2))[:8].tolist())
    assert n >= 25000


def test_emulation_equals_live_cv2_on_frames(emul):
    pytest.importorskip('cv2')
    for img, segs in draw_cases(7, 2, 400, ((720, 1080),)):
        assert np.array_equal(emul_draw(emul, img, segs), cv2_draw(img, segs))


def _digests(lib):
    return [[digest(emul_draw(lib, img, segs)) for img, segs in draw_cases(seed, n, m, sizes)] for seed, n, m, sizes in DIGEST_SETS]


def test_emulation_matches_the_committed_digests(emul):
    doc = json.load(open(DIGESTS))
    assert doc['sets'] == [list(s[:3]) + [[list(x) for x in s[3]]] for s in DIGEST_SETS]
    assert _digests(emul) == doc['digests']


@pytest.mark.parametrize('variant,what', [(1, 'a cap centre one pixel off'), (2, 'the polygon offset truncated, not rounded')])
def test_a_changed_rounding_step_fails_the_digests(variant, what):
    doc = json.load(open(DIGESTS))
    got = _digests(_build(variant))
    wrong = sum(a != b for g, d in zip(got, doc['digests']) for a, b in zip(g, d))
    assert wrong > 0, what


# ---- the planner against the reference's draw_axis ---------------------------------------------------------------------------
def _axis_cases():
    doc = json.load(open(AXIS_JSON))
    z = np.load(AXIS_NPZ)
    for i, case in enumerate(doc['cases']):
        h, w = (int(v) for v in z[f'hw{i}'])
        ang, pts = z[f'ang{i}'], z[f'pts{i}']
        faces = [(*[float(a) for a in ang[k]], pts[k]) for k in range(len(ang))]
        yield i, base_image(i, h, w), faces, case


def _replay(lib, img, faces, plan):
    """draw_axis face after face onto one image; returns (image, name of the exception or None)."""
    canvas = img.copy()
    for yaw, pitch, roll, pts in faces:
        with np.errstate(all='ignore'):
            segs, err = plan(yaw, pitch, roll, pts)
        if segs:
            canvas = emul_draw(lib, canvas, [[x0, y0, x1, y1, c[0] | (c[1] << 8) | (c[2] << 16)] for x0, y0, x1, y1, c in segs])
        if err is not None:
            return canvas, err
    return canvas, None


def test_planner_and_emulation_reproduce_the_reference_draw_axis(emul):
    kinds = {'ValueError': ValueError, 'OverflowError': OverflowError, 'error': OverflowError}   # cv2.error -> OverflowError
    n_err = 0
    for i, img, faces, case in _axis_cases():
        out, err = _replay(emul, img, faces, plan_axis)
        assert digest(out) == case['digest'], i
        assert bool((out != img).any()) == case['changed'], i
        if case['error'] is None:
            assert err is None, (i, err)
        else:
            n_err += 1
            assert type(err) is kinds[case['error']], (i, err, case['error'])
            if case['error'] == 'error':
                assert 'outside int32' in str(err)
    assert n_err == 5


def _plan64(yaw, pitch, roll, pts68):
    """plan_axis with the end points kept in float64 -- what numpy 1's value-based promotion gave."""
    if not all(math.isfinite(a) for a in (yaw, pitch, roll)):
        return plan_axis(yaw, pitch, roll, pts68)
    e = ends64(yaw, pitch, roll, pts68)
    tdx, tdy = float(pts68[0, 30]), float(pts68[1, 30])
    segs = []
    for k, colour in enumerate(AXIS_COLOURS):
        try:
            p0, p1 = (int(tdx), int(tdy)), (int(e[2 * k]), int(e[2 * k + 1]))
        except (ValueError, OverflowError) as err:
            return segs, err
        if not all(-2 ** 31 <= v < 2 ** 31 for v in p0 + p1):
            return segs, OverflowError('outside int32')
        segs.append((*p0, *p1, colour))
    return segs, None


def test_the_golden_cases_tell_float32_from_float64_end_points(emul):
    """The dtype rule is tested, not assumed: a planner that keeps x1 = size * (...) + tdx in float64 gives other bytes on
    some golden cases (the count the golden script recorded has other integer points)."""
    doc = json.load(open(AXIS_JSON))
    differ = sum(digest(_replay(emul, img, faces, _plan64)[0]) != case['digest'] for i, img, faces, case in _axis_cases())
    assert doc['float64_planner_differs'] == 6
    assert differ >= 1, differ


# ---- C entry: argument checks before any CUDA work ----------------------------------------------------------------------------
def _fails(code, want, text):
    assert code == want, (code, _lib.load().syn_last_error())
    assert text in _lib.load().syn_last_error(), _lib.load().syn_last_error()


def test_draw_entry_rejects_bad_arguments():
    lib = _lib.load()
    p = C.c_void_p(8)                                      # never dereferenced: every call below fails validation first
    frames = np.array([[0, 4, 5], [60, 2, 3], [78, 1, 1]], np.int64)
    start = np.array([0, 2, 2, 5], np.int32)

    def draw(img=p, nbytes=81, fr=frames, frd=p, nf=3, st=start, std=p, segs=p, ns=5, th=4, lt=8):
        return lib.syn_draw_lines(img, nbytes, None if fr is None else fr.ctypes.data, frd, nf, None if st is None else st.ctypes.data,
                                  std, segs, ns, th, lt, None)

    _fails(draw(img=None), 1, b'syn_draw_lines: null pointer')
    _fails(draw(fr=None), 1, b'null pointer')
    _fails(draw(frd=None), 1, b'null pointer')
    _fails(draw(st=None), 1, b'null pointer')
    _fails(draw(std=None), 1, b'null pointer')
    _fails(draw(segs=None), 1, b'null pointer')
    _fails(draw(nf=0), 1, b'0 frames')
    _fails(draw(ns=-1), 1, b'-1 segments')
    _fails(draw(nbytes=-1), 1, b'-1 image bytes')
    for th in (1, 2, 3, 5, -1):
        _fails(draw(th=th), 6, b'thickness %d' % th)
    for lt in (4, 16, 0):
        _fails(draw(lt=lt), 6, b'line type %d' % lt)
    for bad, text in (([1, 2, 2, 5], b'must run from 0 to 5'), ([0, 2, 2, 4], b'must run from 0 to 5'),
                      ([0, 3, 2, 5], b'not monotone at frame 1 (2 after 3)')):
        _fails(draw(st=np.array(bad, np.int32)), 4, text)
    _fails(draw(nbytes=80), 4, b'frame 2 (1x1 at byte 78) does not fit the 80 image bytes')
    for bad, text in (([[0, 4, 5], [59, 2, 3], [78, 1, 1]], b'frame 1 (2x3 at byte 59)'),       # overlaps frame 0
                      ([[0, 0, 5], [60, 2, 3], [78, 1, 1]], b'frame 0 is 0x5'),
                      ([[0, 4, 5], [60, 2, -3], [78, 1, 1]], b'frame 1 is 2x-3'),
                      ([[-3, 4, 5], [60, 2, 3], [78, 1, 1]], b'frame 0 (4x5 at byte -3)'),
                      ([[0, 4, 5], [60, 1 << 40, 1 << 40], [78, 1, 1]], b'frame 1 is')):
        _fails(draw(fr=np.array(bad, np.int64)), 4, text)
    # nothing to draw: no launch, no device needed
    assert lib.syn_draw_lines(p, 81, frames.ctypes.data, p, 3, np.zeros(4, np.int32).ctypes.data, p, None, 0, 4, 8, None) == 0


def test_plan_axis_follows_the_reference_failure_order():
    pts = np.zeros((3, 68), np.float32)
    pts[:2] = np.random.default_rng(0).uniform(10, 40, (2, 68))
    segs, err = plan_axis(10.0, 5.0, 0.0, pts)
    assert err is None and [s[4] for s in segs] == list(AXIS_COLOURS) and all(s[:2] == (int(pts[0, 30]), int(pts[1, 30])) for s in segs)
    assert isinstance(plan_axis(float('nan'), 5.0, 0.0, pts)[1], ValueError)
    segs, err = plan_axis(float('inf'), 5.0, 0.0, pts)
    assert segs == [] and isinstance(err, ValueError)
    pts[:2, 30] = 2.0 ** 40
    segs, err = plan_axis(10.0, 5.0, 0.0, pts)
    assert segs == [] and isinstance(err, OverflowError) and 'outside int32' in str(err)
