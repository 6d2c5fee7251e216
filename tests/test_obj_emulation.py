"""CPU checks of the OBJ text without a GPU: tests/host_emul/obj_emul.cpp compiles csrc/obj_math.h -- the header the
CUDA kernels are built from -- with g++.  Its '{:.4f}' field must equal snprintf("%.4f") on every float32 of the
exponents image-space vertices take and on every 4-decimal tie, and Python's str.format on the edge values and on 10^6
random bit patterns; its integer and N.0 fields must equal str.format of int64 and of integral floats; whole files
must equal a Python restatement of the reference's two format strings and the digests of what the reference's own
write_obj / write_obj_with_colors wrote (tests/golden/obj_golden.*).  Also the refusals of the Python writers, which
raise before any CUDA call, and the argument checks of the C entries, which fail before any launch."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from golden.make_golden_obj import edge_values
from synergynet_b200 import _lib, inference
from synergynet_b200.inference import OBJ_NEG_ZERO, ObjTables, obj_field_values, obj_file_name

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_NPZ = os.path.join(HERE, 'golden', 'obj_golden.npz')
GOLDEN_JSON = os.path.join(HERE, 'golden', 'obj_golden.json')


def P(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


@pytest.fixture(scope='module')
def emul():
    out = os.path.join(tempfile.mkdtemp(prefix='obj_emul_'), 'libobj_emul.so')
    subprocess.run(['g++', '-O2', '-shared', '-fPIC', '-pthread', '-o', out, os.path.join(HERE, 'host_emul', 'obj_emul.cpp')],
                   check=True, capture_output=True)
    lib = C.CDLL(out)
    lib.emul_f4.restype = lib.emul_num.restype = lib.emul_f4_sweep.restype = lib.emul_obj.restype = C.c_int64
    lib.emul_f4.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
    lib.emul_num.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
    lib.emul_f4_sweep.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint32)]
    lib.emul_obj.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    return lib


def f4_lines(lib, x):
    x = np.ascontiguousarray(x, np.float32)
    n = lib.emul_f4(P(x), x.size, None)
    out = np.zeros(n, np.uint8)
    assert lib.emul_f4(P(x), x.size, P(out)) == n
    return out.tobytes().decode().split('\n')[:-1]


def num_lines(lib, v, dot0):
    v = np.ascontiguousarray(v, np.int64)
    n = lib.emul_num(P(v), v.size, dot0, None)
    out = np.zeros(n, np.uint8)
    assert lib.emul_num(P(v), v.size, dot0, P(out)) == n
    return out.tobytes().decode().split('\n')[:-1]


def python_f4(x):
    return ['{:.4f}'.format(v) for v in np.asarray(x, np.float32)]


# ---- the '{:.4f}' field --------------------------------------------------------------------------------------------------
def test_f4_edge_values_equal_python(emul):
    e = edge_values()
    got = f4_lines(emul, e)
    assert got == python_f4(e)
    by_value = dict(zip(np.asarray(e).view(np.uint32).tolist(), got))
    assert by_value[0x80000000] == '-0.0000' and by_value[0xFFC00000] == 'nan' and by_value[0xFF800000] == '-inf'
    assert by_value[0x7F7FFFFF] == '{:.4f}'.format(np.finfo(np.float32).max) and len(by_value[0x7F7FFFFF]) == 44
    assert f4_lines(emul, [0.03125, 0.09375, -1e-5, 1e20]) == ['0.0312', '0.0938', '-0.0000', '100000002004087734272.0000']


def test_f4_random_bit_patterns_equal_python(emul):
    rng = np.random.default_rng(1)
    x = rng.integers(0, 1 << 32, 1 << 20, dtype=np.uint64).astype(np.uint32).view(np.float32)
    assert f4_lines(emul, x) == python_f4(x)


@pytest.mark.parametrize('be_lo,be_hi', [(112, 124), (125, 137), (138, 150)])
def test_f4_every_mantissa_of_the_vertex_exponents_equals_snprintf(emul, be_lo, be_hi):
    """|x| in [2^-15, 2^24), both signs, every mantissa: biased exponents 112..150."""
    first = C.c_uint32(0)
    bad = emul.emul_f4_sweep(be_lo, be_hi, 0, C.byref(first))
    assert bad == 0, (bad, hex(first.value))


def test_f4_every_tie_equals_snprintf(emul):
    """The odd multiples of 2^-5 float32 holds, both signs: exactly the values whose 4-decimal rounding is a tie."""
    first = C.c_uint32(0)
    assert emul.emul_f4_sweep(0, 0, 1, C.byref(first)) == 0, hex(first.value)
    ties = (2 * np.arange(0, 1 << 23, 4099, dtype=np.float64) + 1) / 32
    assert f4_lines(emul, ties) == python_f4(ties)


# ---- the '{}' fields -----------------------------------------------------------------------------------------------------------
def test_integer_field_equals_python(emul):
    v = np.array([0, 1, -1, 9, 10, -10, 99, 100, 53214, 2 ** 31 - 1, -2 ** 31, 2 ** 63 - 1, -2 ** 63, -2 ** 63 + 1, 10 ** 18,
                  -10 ** 18, 999999999999999999], np.int64)
    v = np.concatenate([v, np.random.default_rng(2).integers(-2 ** 63, 2 ** 63 - 1, 20000, dtype=np.int64)])
    assert num_lines(emul, v, 0) == ['{}'.format(x) for x in v]


def test_n0_field_equals_python_below_1e16(emul):
    f = np.array([0.0, -0.0, 1.0, -1.0, 233.0, 255.0, 2.0 ** 53, 9999999999999998.0, -9999999999999998.0, 1e15, 12345678.0],
                 np.float64)
    f = np.concatenate([f, np.random.default_rng(3).integers(-10 ** 16 + 1, 10 ** 16, 20000).astype(np.float64)])
    v, dot0 = obj_field_values(f, 'f')
    assert dot0 == 1 and v[1] == OBJ_NEG_ZERO
    assert num_lines(emul, v, 1) == ['{}'.format(x) for x in f]
    f32 = np.arange(256, dtype=np.float32)
    assert num_lines(emul, obj_field_values(f32, 'c')[0], 1) == ['{}'.format(x) for x in f32]
    assert num_lines(emul, obj_field_values(np.array([-0.0], np.float32), 'c')[0], 1) == ['-0.0']


@pytest.mark.parametrize('bad', [1e16, -1e16, 2.0 ** 60, 0.5, -233.25, float('nan'), float('inf'), float('-inf')])
def test_n0_field_refuses_what_needs_shortest_round_trip(bad):
    a = np.array([1.0, 2.0, bad, 3.0])
    with pytest.raises(ValueError, match=r'\[2\] = '):
        obj_field_values(a, 'colors')
    with pytest.raises(ValueError, match='triangles'):
        ObjTables(np.array([[1.0, 2.0], [3.0, bad], [4.0, 5.0]]), 10)


def test_file_names():
    assert [obj_file_name(n) for n in ('mesh', 'mesh.obj', 'a.b', 'x.OBJ', 'y.', 'z.obj.obj', 'dir.obj/face')] == \
        ['mesh.obj', 'mesh.obj', 'a.b.obj', 'x.OBJ.obj', 'y..obj', 'z.obj.obj', 'dir.obj/face.obj']


# ---- whole files ----------------------------------------------------------------------------------------------------------------
def emul_file(lib, vertices, triangles, colors=None, keep=None):
    """The bytes the kernels write for one mesh, from the same host tables the Python writers build."""
    t = ObjTables(triangles, vertices.shape[1], colors, keep, 1)
    xyz = np.ascontiguousarray(vertices.T if keep is None else vertices[:, keep].T, np.float32)
    col = None if t.colors is None else np.ascontiguousarray(t.colors[0])
    tri = np.ascontiguousarray(t.tri)
    args = (P(xyz), xyz.shape[0], P(col), t.colors_dot0, P(tri), tri.shape[0], 0 if col is None else 1, t.tri_dot0)
    n = lib.emul_obj(*args, None)
    out = np.zeros(n, np.uint8)
    assert lib.emul_obj(*args, P(out)) == n
    return out.tobytes()


def python_obj(vertices, triangles, colors=None):
    """The two reference format strings, restated."""
    s = []
    for i in range(vertices.shape[1]):
        if colors is None:
            s.append('v {:.4f} {:.4f} {:.4f}\n'.format(vertices[0, i], vertices[1, i], vertices[2, i]))
        else:
            s.append('v {:.4f} {:.4f} {:.4f} {} {} {}\n'.format(vertices[0, i], vertices[1, i], vertices[2, i], colors[i, 2],
                                                               colors[i, 1], colors[i, 0]))
    for i in range(triangles.shape[1]):
        order = (2, 1, 0) if colors is None else (0, 1, 2)
        s.append('f {} {} {}\n'.format(*(triangles[k, i] for k in order)))
    return ''.join(s).encode()


def golden_cases():
    doc = json.load(open(GOLDEN_JSON))
    z = np.load(GOLDEN_NPZ)
    for i, case in enumerate(doc['cases']):
        v, tri = z[f'vertices{i}'], z[f'triangles{i}']
        if case['kind'] == 'obj':
            yield case, (v, tri, None, None)
        else:
            keep = z[f'keep{i}']
            col = z[f'colors_u8{i}'][keep]
            yield case, (v, tri, col.astype(np.float32) if z[f'colors_f32{i}'][0] else col, keep)


def test_emulated_files_equal_the_reference_digests(emul):
    n = 0
    for case, (v, tri, col, keep) in golden_cases():
        data = emul_file(emul, v, tri, col, keep)
        assert len(data) == case['bytes'] and hashlib.sha256(data).hexdigest() == case['sha256'], case
        assert obj_file_name(case['name']) == case['written']
        n += 1
    assert n == 7


def test_emulated_files_equal_the_format_strings(emul):
    rng = np.random.default_rng(4)
    for trial in range(6):
        n, ntri = int(rng.integers(1, 400)), int(rng.integers(0, 300))
        v = (rng.normal(0, 10 ** rng.uniform(-3, 6), (3, n))).astype(np.float32)
        v.reshape(-1)[rng.integers(0, v.size, 5)] = edge_values()[rng.integers(0, edge_values().size, 5)]
        tri = rng.integers(-5, 10 ** 9, (3, ntri)).astype([np.int32, np.int64, np.float64][trial % 3])
        assert emul_file(emul, v, tri) == python_obj(v, tri)
        keep = np.sort(rng.choice(n, max(1, n // 2), replace=False))
        col = rng.integers(0, 256, (len(keep), 3)).astype([np.uint8, np.float32][trial % 2])
        assert emul_file(emul, v, tri, col, keep) == python_obj(v[:, keep], tri, col)


# ---- refusals before any CUDA call ----------------------------------------------------------------------------------------------
@pytest.fixture
def no_cuda(monkeypatch):
    import torch

    def touched(*a, **k):
        raise AssertionError('a refused call reached CUDA')
    monkeypatch.setattr(torch.cuda, 'is_available', touched)
    monkeypatch.setattr(inference, 'obj_encoder', touched)
    monkeypatch.setattr(inference, '_obj_upload', touched)


def test_writers_refuse_before_cuda(no_cuda, tmp_path):
    import torch
    v = np.zeros((3, 10), np.float32)
    tri = np.array([[1], [2], [3]])
    col = np.zeros((10, 3), np.uint8)
    name = str(tmp_path / 'm')
    cases = [
        (TypeError, lambda: inference.write_obj(name, v.astype(np.float64), tri)),
        (TypeError, lambda: inference.write_obj(name, torch.zeros((3, 10), dtype=torch.float64), tri)),
        (ValueError, lambda: inference.write_obj(name, np.zeros((4, 10), np.float32), tri)),
        (ValueError, lambda: inference.write_obj(name, np.zeros((3, 0), np.float32), tri)),
        (ValueError, lambda: inference.write_obj(name, v, tri.T)),
        (ValueError, lambda: inference.write_obj(name, v, tri.astype(np.float64) + 0.5)),
        (TypeError, lambda: inference.write_obj(name, v, tri.astype(bool))),
        (ValueError, lambda: inference.write_obj_with_colors(name, v, tri, col.astype(np.float32) + 0.25)),
        (ValueError, lambda: inference.write_obj_with_colors(name, v, tri, col[:9])),
        (ValueError, lambda: inference.write_obj_with_colors(name, v, tri, np.full((10, 3), 1e16))),
        (ValueError, lambda: inference.obj_bytes(v, tri, keep=np.array([0, 10]))),
        (ValueError, lambda: inference.obj_bytes(v, tri, keep=np.array([-1]))),
        (ValueError, lambda: inference.obj_bytes(np.zeros((2, 3, 10), np.float32), tri, np.zeros((3, 10, 3), np.uint8))),
    ]
    for kind, call in cases:
        with pytest.raises(kind):
            call()
    assert not list(tmp_path.iterdir())


# ---- C entries: argument checks before any launch -------------------------------------------------------------------------------
def _fails(code, want, text):
    assert code == want, (code, _lib.load().syn_last_error())
    assert text in _lib.load().syn_last_error(), _lib.load().syn_last_error()


def test_obj_entries_reject_bad_arguments():
    lib = _lib.load()
    p = 8                                                   # never dereferenced: every call below fails validation first
    keep = np.array([0, 5, 9], np.int32)

    def desc(**kw):
        d = _lib.ObjDesc(vertices=p, stride_mesh=30, stride_vertex=1, stride_coord=10, batch=2, nver=10, keep_host=None,
                         keep_dev=None, n_keep=0, colors=None, colors_stride_mesh=0, colors_dot0=0, triangles=p, ntri=4,
                         tri_order=0, tri_dot0=0)
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    ws = int(lib.syn_obj_workspace_size(2, 10, 4))
    assert ws == 8 * (1 + 2 + 1)
    assert lib.syn_obj_workspace_size(0, 10, 4) == -1 and lib.syn_obj_workspace_size(1, -1, 4) == -1
    assert lib.syn_obj_workspace_size(65536, 10, 4) == -1 and lib.syn_obj_workspace_size(65535, 2 ** 31 - 1, 0) == -1
    assert lib.syn_obj_workspace_size(65535, 10, 4) == 8 * (1 + 65535 + 1)

    def both(d, code, text, ws_bytes=ws):
        _fails(lib.syn_obj_plan(C.byref(d), p, ws_bytes, p, None), code, text)
        assert lib.syn_last_error().startswith(b'syn_obj_plan: ')
        _fails(lib.syn_obj_write(C.byref(d), p, ws_bytes, p, p, 100, None), code, text)
        assert lib.syn_last_error().startswith(b'syn_obj_write: ')

    _fails(lib.syn_obj_plan(None, p, ws, p, None), 1, b'null pointer')
    both(desc(vertices=None), 1, b'null pointer')
    both(desc(triangles=None), 1, b'null pointer')
    both(desc(keep_host=keep.ctypes.data, n_keep=3), 1, b'null pointer')
    both(desc(keep_dev=p, n_keep=3), 1, b'keep_dev without keep_host')
    both(desc(batch=65535, nver=2 ** 31 - 1), 1, b"65535 meshes of 2147483647 vertex lines and 4 triangles exceed one launch's")
    _fails(lib.syn_obj_plan(C.byref(desc()), None, ws, p, None), 1, b'null pointer')
    _fails(lib.syn_obj_plan(C.byref(desc()), p, ws, None, None), 1, b'null pointer')
    _fails(lib.syn_obj_write(C.byref(desc()), p, ws, None, p, 100, None), 1, b'null pointer')
    _fails(lib.syn_obj_write(C.byref(desc()), p, ws, p, None, 100, None), 1, b'null pointer')
    _fails(lib.syn_obj_write(C.byref(desc()), p, ws, p, p, -1, None), 1, b'-1 output bytes')
    for kw, text in ((dict(batch=0), b'0 meshes'), (dict(batch=-3), b'-3 meshes'), (dict(batch=65536), b'65536 meshes'),
                     (dict(nver=0), b'0 vertices'), (dict(ntri=-1), b'-1 triangles'),
                     (dict(keep_host=keep.ctypes.data, keep_dev=p, n_keep=-2), b'-2 kept')):
        both(desc(**kw), 1, text)
    for kw in (dict(stride_vertex=0), dict(stride_coord=-1), dict(stride_mesh=0), dict(colors_stride_mesh=-3)):
        both(desc(**kw), 1, b'strides')
    for kw in (dict(tri_order=2), dict(tri_dot0=-1), dict(colors_dot0=3)):
        both(desc(**kw), 1, b'flags')
    for bad, at in (([0, 10, 3], 1), ([-1], 0), ([2, 3, 4, 2 ** 31 - 1], 3)):
        k = np.array(bad, np.int32)
        both(desc(keep_host=k.ctypes.data, keep_dev=p, n_keep=len(bad)), 1, b'keep[%d] = %d lies outside [0, 10)' % (at, bad[at]))
    both(desc(), 4, b'workspace of 31 bytes, 32 needed', ws_bytes=31)
    _fails(lib.syn_obj_plan(C.byref(desc(batch=1, stride_mesh=0)), p, 23, p, None), 4, b'23 bytes, 24 needed')   # one mesh: any stride_mesh
