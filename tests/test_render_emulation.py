"""CPU checks of the render / NMS kernels' arithmetic and algorithms without a GPU: tests/host_emul/render_emul.cpp
compiles csrc/render_math.h -- the header the CUDA kernels are built from -- with g++ and runs the kernels' algorithms
(incidence-list normals, key-maximum z-buffer, bit-matrix NMS) as serial loops.  They must return the oracle's bits.
Also covers the host-side entry points of the C ABI for this stage (incidence lists, argument validation)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import render_cases as rc
from oracle import render_port as rp
from synergynet_b200 import _lib, synthetic

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, 'golden', 'render_vectors.npz')


def P(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope='module')
def emul():
    out = os.path.join(tempfile.mkdtemp(prefix='render_emul_'), 'librender_emul.so')
    subprocess.run(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', out, os.path.join(HERE, 'host_emul', 'render_emul.cpp')],
                   check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.emul_nms.restype = C.c_int
    return lib


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLD, allow_pickle=False))


def incidence(tri, nver):
    lib = _lib.load()
    start = np.zeros(nver + 1, np.int32)
    lst = np.zeros(tri.size, np.int32)
    _lib.check(lib.syn_mesh_incidence_host(tri.ctypes.data, tri.shape[0], nver, start.ctypes.data, lst.ctypes.data))
    return start, lst


def light_cfg():
    v3 = lambda *x: (C.c_float * 3)(*x)
    return _lib.LightCfg(0.75, 0.7, 0.2, v3(1, 1, 1), v3(1, 1, 1), v3(0, 0, 5), v3(0, 0, 5), 5)


def test_incidence_lists():
    tri = np.array([[0, 1, 2], [2, 1, 3], [3, 3, 0], [1, 0, 2]], np.int32)
    start, lst = incidence(tri, 5)
    assert start.tolist() == [0, 3, 6, 9, 12, 12]                       # vertex 4 is isolated
    per = [lst[start[v]:start[v + 1]].tolist() for v in range(5)]
    assert per == [[0, 2, 3], [0, 1, 3], [0, 1, 3], [1, 2, 2], []]       # ascending; a repeated corner is listed twice
    bad = np.array([[0, 1, 7]], np.int32)
    rc = _lib.load().syn_mesh_incidence_host(bad.ctypes.data, 1, 5, start.ctypes.data, lst.ctypes.data)
    assert rc == 4                                                        # SYN_ERR_SHAPE


def test_normals_and_lighting(emul, gold):
    tri, verts = gold['render_tri'], gold['render_verts']
    n = verts.shape[2]
    start, lst = incidence(tri, n)
    cfg = light_cfg()
    for b in range(verts.shape[0]):
        plane = np.ascontiguousarray(verts[b])                             # (3,N): stride_vertex 1, stride_coord N
        inter = np.ascontiguousarray(verts[b].T)                           # (N,3): stride_vertex 3, stride_coord 1
        for arr, sv, sc in ((plane, 1, n), (inter, 3, 1)):
            out = np.zeros((n, 3), np.float32)
            emul.emul_normals(P(arr), sv, sc, n, P(tri), tri.shape[0], P(start), P(lst), P(out))
            assert np.array_equal(out, gold['render_normals'][b])
            light = np.zeros((n, 3), np.float32)
            emul.emul_lighting(P(arr), sv, sc, n, P(out), C.byref(cfg), None, P(light))
            assert np.abs(light - gold['render_light'][b]).max() <= 2e-7
            tex = np.random.default_rng(b).uniform(0, 1, (n, 3)).astype(np.float32)
            lt = np.zeros((n, 3), np.float32)
            emul.emul_lighting(P(arr), sv, sc, n, P(out), C.byref(cfg), P(tex), P(lt))
            assert np.array_equal(lt, tex * light)


def test_isolated_vertex_is_nan_like_the_reference(emul):
    tri = np.array([[0, 1, 2]], np.int32)
    ver = np.array([[0, 0, 0], [4, 0, 1], [0, 4, 2], [9, 9, 9]], np.float32)
    start, lst = incidence(tri, 4)
    out = np.zeros((4, 3), np.float32)
    emul.emul_normals(P(ver), 3, 1, 4, P(tri), 1, P(start), P(lst), P(out))
    assert np.array_equal(out, rp.get_normal(ver, tri), equal_nan=True) and np.isnan(out[3]).all()


@pytest.mark.parametrize('shuffle', [0, 1])
def test_rasterize_batch_bit_exact(emul, gold, shuffle):
    tri, verts, bg = gold['render_tri'], gold['render_verts'], gold['render_bg']
    b, _, n = verts.shape
    h, w, c = bg.shape
    colors = np.ascontiguousarray(gold['render_light'])
    img = bg.copy()
    depth = np.zeros((b, h, w), np.float32)
    emul.emul_rasterize(P(img), h, w, c, P(verts), C.c_longlong(3 * n), 1, n, b, n, P(tri), tri.shape[0], P(colors),
                        C.c_float(1.0), 0, P(depth), shuffle)
    assert np.array_equal(img, gold['render_steps'][-1])                   # the reference after its third mesh
    for k in range(b):
        _, d = rp.rasterize(np.ascontiguousarray(verts[k].T), tri, colors[k], bg.copy(), return_depth=True)
        assert np.array_equal(depth[k], d)
    # single mesh, reverse
    img = bg.copy()
    v0 = np.ascontiguousarray(verts[0].T)
    emul.emul_rasterize(P(img), h, w, c, P(v0), C.c_longlong(0), 3, 1, 1, n, P(tri), tri.shape[0], P(gold['raster_colors']),
                        C.c_float(1.0), 1, None, shuffle)
    assert np.array_equal(img, gold['raster_reverse'])


def test_rasterize_ties_and_large_triangles(emul):
    """Coplanar duplicates (depth ties: the first triangle must win), triangles larger than the image, triangles wholly
    outside, zero-area triangles."""
    ver = np.array([[-30, -20, 1], [90, -10, 1], [20, 100, 1],            # huge, constant depth
                    [5, 5, 1], [40, 8, 1], [12, 50, 1],                   # inside the first, same depth -> tie
                    [200, 200, 5], [210, 200, 5], [200, 210, 5],          # outside
                    [10, 10, 3], [10, 10, 3], [30, 30, 3]], np.float32)   # degenerate
    tri = np.array([[0, 1, 2], [3, 4, 5], [0, 1, 2], [6, 7, 8], [9, 10, 11], [5, 4, 3]], np.int32)
    col = np.random.default_rng(0).uniform(0, 1, (12, 3)).astype(np.float32)
    bg = np.full((48, 64, 3), 17, np.uint8)
    want, dwant = rp.rasterize(ver, tri, col, bg.copy(), return_depth=True)
    for shuffle in (0, 1):
        img = bg.copy()
        depth = np.zeros((1, 48, 64), np.float32)
        emul.emul_rasterize(P(img), 48, 64, 3, P(ver), C.c_longlong(0), 3, 1, 1, 12, P(tri), 6, P(col), C.c_float(1.0), 0, P(depth), shuffle)
        assert np.array_equal(img, want) and np.array_equal(depth[0], dwant)
    assert (want != 17).any()


def test_rasterize_signed_zero_depth_tie(emul):
    """Two coplanar copies of one triangle at depth -0 and then +0: the reference's serial `>` sees a tie, so the FIRST
    triangle's colour stays, whatever order the order-free key processes them in."""
    xy = [[2, 2], [30, 3], [6, 25]]
    ver = np.array([p + [-0.0] for p in xy] + [p + [0.0] for p in xy], np.float32)
    tri = np.array([[0, 1, 2], [3, 4, 5]], np.int32)
    col = np.array([[0.9, 0.1, 0.1]] * 3 + [[0.1, 0.1, 0.9]] * 3, np.float32)
    bg = np.zeros((32, 32, 3), np.uint8)
    want, dwant = rp.rasterize(ver, tri, col, bg.copy(), return_depth=True)
    assert (want[..., 0] == 229).any() and not (want[..., 2] == 229).any()    # the reference keeps the first triangle
    for shuffle in (0, 1):
        img = bg.copy()
        depth = np.zeros((1, 32, 32), np.float32)
        emul.emul_rasterize(P(img), 32, 32, 3, P(ver), C.c_longlong(0), 3, 1, 1, 6, P(tri), 2, P(col), C.c_float(1.0), 0, P(depth), shuffle)
        assert np.array_equal(img, want) and np.array_equal(depth[0], dwant)


OOR = rc.out_of_range_cases()


@pytest.mark.parametrize('case', OOR, ids=[c[0] for c in OOR])
def test_rasterize_out_of_range_values(emul, case):
    """Coordinates at and beyond 2^31, infinities and NaN, depths at the buffer's initial -1e8, colours whose byte wraps
    or overflows int, degenerate triangles: render_math.h's conversions must give the reference's x86 results (a far
    vertex skips its triangle, an overflowing colour writes 0), bit for bit with the port and the reference itself."""
    _, ver, tri, col = case
    h, w = rc.CANVAS
    bg = np.random.default_rng(len(case[0])).integers(0, 256, (h, w, 3), dtype=np.uint8)
    for reverse in (False, True):
        want, dwant = rp.rasterize(ver, tri, col, bg.copy(), reverse=reverse, return_depth=True)
        if rp.have_ref():
            ref, dref = rp.rasterize(ver, tri, col, bg.copy(), reverse=reverse, return_depth=True, kind='ref')
            assert np.array_equal(ref, want) and np.array_equal(dref, dwant)
        for shuffle in (0, 1):
            img = bg.copy()
            depth = np.zeros((1, h, w), np.float32)
            emul.emul_rasterize(P(img), h, w, 3, P(ver), C.c_longlong(0), 3, 1, 1, ver.shape[0], P(tri), tri.shape[0], P(col),
                                C.c_float(1.0), int(reverse), P(depth), shuffle)
            assert np.array_equal(img, want) and np.array_equal(depth[0], dwant)
        assert (want != bg).any()                                   # the ordinary triangle of every case is drawn


def test_out_of_range_cases_separate_x86_from_saturation():
    """The cases hold the values where x86's conversion and a saturating one part: a far vertex skips its triangle, an
    overflowing colour is written as 0."""
    h, w = rc.CANVAS
    names = {c[0]: c for c in OOR}
    bg = np.zeros((h, w, 3), np.uint8)
    _, ver, tri, col = names['vertex_x=3e+09']
    assert not rc.tri_boxes(ver, tri, h, w)[1][0]
    alone = rp.rasterize(ver, tri[:1], col, bg.copy())
    assert not alone.any()                                          # a saturating conversion would draw 640 pixels
    for tag in ('8421505', '1e10', 'inf'):
        _, ver, tri, col = names[f'colour={tag}']
        img, d = rp.rasterize(ver, tri[:1], col, bg.copy(), return_depth=True)
        assert (d > -1e8).sum() > 100 and (img[..., 0][d > -1e8] == 0).mean() > 0.5, tag
    _, ver, tri, col = names['colour=8421504']
    img, d = rp.rasterize(ver, tri[:1], col, bg.copy(), return_depth=True)
    assert (img[..., 0][d > -1e8] == 128).any()                     # 255 * 8421504 = 2^31 - 128: converts, low byte 0x80
    assert np.array_equal(rc.x86_int(np.array([rc.F_BELOW_2_31, 2.0 ** 31, -2.0 ** 31, np.nan, -np.inf, -1.5], np.float32)),
                          [2 ** 31 - 128, rc.INT_MIN, rc.INT_MIN, rc.INT_MIN, rc.INT_MIN, -1])


def test_nms_bitmatrix_equals_greedy(emul, gold):
    d = gold['nms_dets']
    order = d[:, 4].argsort()[::-1]
    ds = np.ascontiguousarray(d[order])
    keep = np.zeros(ds.shape[0], np.int32)
    for thr, key in ((0.3, 'nms_keep_3'), (0.5, 'nms_keep_5')):
        for ge in (0, 1):
            n = emul.emul_nms(P(ds), ds.shape[0], C.c_double(thr), ge, P(keep))
            assert order[keep[:n]].tolist() == gold[key].tolist()
    # equality at the threshold separates the two conventions
    two = np.array([[0, 0, 9, 9, 0.9], [5, 0, 14, 9, 0.8]], np.float32)
    thr = float(np.float32(50.0) / np.float32(150.0))
    assert emul.emul_nms(P(two), 2, C.c_double(thr), 1, P(keep)) == 1
    assert emul.emul_nms(P(two), 2, C.c_double(thr), 0, P(keep)) == 2


def test_cabi_argument_checks():
    lib = _lib.load()
    assert lib.syn_faceboxes_num_priors(250, 333) == rp.prior_boxes(250, 333).shape[0]
    assert lib.syn_faceboxes_num_priors(720, 1080) == 21 * 23 * 34 + 12 * 17 + 6 * 9
    assert lib.syn_faceboxes_num_priors(0, 5) == -1
    one = C.c_void_p(8)     # never dereferenced: the calls below fail validation before any CUDA work
    # alpha != 1 has no order-free result: refused, not approximated
    rc = lib.syn_rasterize(one, 8, 8, 3, one, 24, 3, 1, 1, 8, one, 1, one, C.c_float(0.5), 0, one, None, None)
    assert rc == 6 and b'alpha' in lib.syn_last_error()
    assert lib.syn_rasterize(None, 8, 8, 3, one, 24, 3, 1, 1, 8, one, 1, one, C.c_float(1.0), 0, one, None, None) == 1
    assert lib.syn_mesh_normals(one, 24, 0, 1, 1, 8, one, 1, one, one, one, one, None) == 1      # zero vertex stride
    assert lib.syn_nms(one, 4, C.c_double(0.3), 7, one, one, one, None) == 1                       # unknown mode


def test_product_modules_fail_loudly_without_a_gpu():
    """No CPU fallback in the Sim3DR / FaceBoxes modules: without a CUDA device every entry raises instead of computing."""
    import torch
    if torch.cuda.is_available():
        pytest.skip('this host has a GPU')
    from synergynet_b200 import Sim3DR, detect, faceboxes
    tri = np.array([[0, 1, 2]], np.int32)
    ver = np.zeros((3, 3), np.float32)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        Sim3DR.get_normal(ver, tri)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        Sim3DR.rasterize(ver, tri, ver, bg=np.zeros((4, 4, 3), np.uint8))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        detect.nms(np.zeros((2, 5), np.float32), 0.3)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0))
    assert detect.nms(np.zeros((0, 5), np.float32), 0.3) == []            # nms_wrapper.py:16-17 needs no device


# ---- property tests: random meshes / boxes through the kernels' algorithms vs the oracle ---------------------------------------
from hypothesis import given, settings, strategies as st  # noqa: E402


@settings(max_examples=40, deadline=None)
@given(seed=st.integers(0, 10_000), nver=st.integers(3, 40), ntri=st.integers(1, 60), h=st.integers(1, 40), w=st.integers(1, 48),
       spread=st.sampled_from([0.5, 1.0, 3.0]), quantise=st.booleans(), reverse=st.booleans())
def test_rasterizer_algorithm_on_random_meshes(emul, seed, nver, ntri, h, w, spread, quantise, reverse):
    """Random triangles -- partly or wholly outside the image, sliver and zero-area ones, integer coordinates that put
    pixel centres exactly on edges and make depth ties -- in natural and scrambled order: image and depth buffer must be
    the serial reference's, bit for bit."""
    rng = np.random.default_rng(seed)
    ver = np.stack([rng.uniform(-spread * w * 0.3, w * (1 + 0.3 * spread), nver), rng.uniform(-spread * h * 0.3, h * (1 + 0.3 * spread), nver),
                    rng.uniform(-5, 5, nver)], 1).astype(np.float32)
    if quantise:
        ver = np.round(ver)
    tri = rng.integers(0, nver, (ntri, 3)).astype(np.int32)
    col = rng.uniform(0, 1, (nver, 3)).astype(np.float32)
    bg = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    want, dwant = rp.rasterize(ver, tri, col, bg.copy(), reverse=reverse, return_depth=True)
    for shuffle in (0, 1):
        img = bg.copy()
        depth = np.zeros((1, h, w), np.float32)
        emul.emul_rasterize(P(img), h, w, 3, P(ver), C.c_longlong(0), 3, 1, 1, nver, P(tri), ntri, P(col), C.c_float(1.0), int(reverse),
                            P(depth), shuffle)
        assert np.array_equal(img, want) and np.array_equal(depth[0], dwant)


@settings(max_examples=40, deadline=None)
@given(seed=st.integers(0, 10_000), nver=st.integers(3, 30), ntri=st.integers(1, 80))
def test_normals_algorithm_on_random_topologies(emul, seed, nver, ntri):
    """Random triangle lists (repeated corners, isolated vertices -> NaN like the reference) through the incidence-list sum."""
    rng = np.random.default_rng(seed)
    ver = rng.normal(0, 10, (nver, 3)).astype(np.float32)
    tri = rng.integers(0, nver, (ntri, 3)).astype(np.int32)
    start, lst = incidence(tri, nver)
    out = np.zeros((nver, 3), np.float32)
    emul.emul_normals(P(ver), 3, 1, nver, P(tri), ntri, P(start), P(lst), P(out))
    assert np.array_equal(out, rp.get_normal(ver, tri), equal_nan=True)


@settings(max_examples=40, deadline=None)
@given(seed=st.integers(0, 10_000), n=st.integers(1, 300), grid=st.sampled_from([1.0, 4.0, 16.0]), thr=st.sampled_from([0.3, 0.5, 1.0 / 3.0]))
def test_nms_algorithm_on_random_boxes(emul, seed, n, grid, thr):
    """Boxes snapped to a grid (many overlaps are exact small fractions, some equal to the threshold) through the bit-matrix
    + block scan, both comparison conventions, vs the serial C restatement and numpy's py_cpu_nms."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(0, 200, (n, 2))
    wh = rng.uniform(8, 90, (n, 2))
    d = np.hstack([np.round((c - wh / 2) / grid) * grid, np.round((c + wh / 2) / grid) * grid, (rng.permutation(n)[:, None] + 1.0) / (n + 1)])
    d = d.astype(np.float32)
    order = d[:, 4].argsort()[::-1]
    ds = np.ascontiguousarray(d[order])
    keep = np.zeros(n, np.int32)
    for ge in (1, 0):
        k = emul.emul_nms(P(ds), n, C.c_double(thr), ge, P(keep))
        assert order[keep[:k]].tolist() == rp.cpu_nms(d, thr, ge=bool(ge))
    k = emul.emul_nms(P(ds), n, C.c_double(thr), 0, P(keep))
    assert order[keep[:k]].tolist() == rp.py_cpu_nms(d, np.float32(thr))
