"""The OBJ text on the H100: syn_obj_plan / syn_obj_write against the host emulation of the same header (which
test_obj_emulation.py holds to Python's str.format), write_obj / write_obj_with_colors against the reference's own
files (the committed golden digests), and the models' obj_batch / obj_images against get_all_outputs_* followed by the
per-face write_obj they replace.  Every equality is byte for byte."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import synth_mbv1, synth_model, synth_resnet
from oracle.stage_check import make_model
from synergynet_b200 import _lib, synthetic
from synergynet_b200.inference import ObjTables, obj_bytes, obj_encoder, write_obj, write_obj_with_colors
from test_obj_emulation import emul, emul_file, golden_cases, python_obj  # noqa: F401  (emul is a fixture)

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)


def _meshes(rng, b, n, edge=True):
    """(b,3,n) float32 image-space meshes, the first carrying special values."""
    v = np.stack([rng.uniform(-20, 700, (b, n)), rng.uniform(-20, 500, (b, n)), rng.normal(0, 60, (b, n))], 1).astype(np.float32)
    if edge:
        from golden.make_golden_obj import edge_values
        e = edge_values()[:n]
        v[0, 1, :e.size] = e
    return v


def test_writers_equal_the_reference_files(tmp_path):
    for k, (case, (v, tri, col, keep)) in enumerate(golden_cases()):
        for on_device in (False, True):
            vv = torch.from_numpy(v).to(DEV) if on_device else v
            name = str(tmp_path / f'{k}{int(on_device)}_{case["name"]}')
            if col is None:
                write_obj(name, vv, tri)
            else:
                write_obj_with_colors(name, vv[:, keep] if on_device else v[:, keep], tri, col)
            (f,) = list(tmp_path.iterdir())
            assert f.name == f'{k}{int(on_device)}_{case["written"]}'
            data = f.read_bytes()
            f.unlink()
            assert hashlib.sha256(data).hexdigest() == case['sha256'], (k, on_device)


@pytest.mark.parametrize('b,n,ntri', [(1, 1, 0), (1, 255, 1), (3, 257, 513), (5, 1000, 77), (2, 53215, 105840)])
def test_batches_equal_the_emulation(emul, b, n, ntri):  # noqa: F811
    rng = np.random.default_rng(b * 7 + n)
    v = _meshes(rng, b, n)
    tri = rng.integers(1, n + 1, (3, ntri))
    got = obj_bytes(torch.from_numpy(v).to(DEV), tri)
    assert len(got) == b
    for i in range(b):
        assert got[i] == emul_file(emul, v[i], tri), i
    if n < 2000:
        assert got[0] == python_obj(v[0], tri)


def test_strided_views_keep_and_colours(emul):  # noqa: F811
    rng = np.random.default_rng(3)
    b, n = 4, 700
    rows = torch.from_numpy(_meshes(rng, b, n).transpose(0, 2, 1).copy()).to(DEV)          # (B,N,3) storage
    v = rows.transpose(1, 2)                                                              # (B,3,N) view, strides (3N,1,3)
    host = v.cpu().numpy()
    tri = rng.integers(1, 300, (3, 411)).astype(np.float64)
    keep = np.sort(rng.choice(n, 299, replace=False))
    shared = rng.integers(0, 256, (299, 3)).astype(np.uint8)
    per_mesh = rng.integers(0, 256, (b, 299, 3)).astype(np.float32)
    assert obj_bytes(v, tri) == [emul_file(emul, host[i], tri) for i in range(b)]
    assert obj_bytes(v, tri, keep=keep) == [emul_file(emul, host[i][:, keep], tri) for i in range(b)]
    assert obj_bytes(v, tri, shared, keep) == [emul_file(emul, host[i], tri, shared, keep) for i in range(b)]
    assert obj_bytes(v, tri, per_mesh, keep) == [emul_file(emul, host[i], tri, per_mesh[i], keep) for i in range(b)]
    assert obj_bytes(v, tri, torch.from_numpy(per_mesh).to(DEV), keep)[2] == python_obj(host[2][:, keep], tri, per_mesh[2])
    one = rows[1]                                                                         # an (nver,3) array
    assert obj_bytes(one.T, tri) == [emul_file(emul, host[1], tri)]


def test_chunks_and_stale_memory(emul):  # noqa: F811
    """Many small chunks equal one pass; a call after a larger one (stale workspace) and an output poisoned with 0xFF give
    the same bytes."""
    rng = np.random.default_rng(4)
    v = torch.from_numpy(_meshes(rng, 9, 3001)).to(DEV)
    tri = rng.integers(1, 3001, (3, 2000))
    t = ObjTables(tri, 3001)
    whole = t.encode(v)
    assert t.encode(v, chunk_bytes=300_000) == whole                                       # 2 meshes per chunk
    assert whole == [emul_file(emul, v[i].cpu().numpy(), tri) for i in range(9)]
    small = v[3:5]
    d = t.desc(small, 0, DEV)
    enc = obj_encoder(DEV)
    ws = enc.workspace(2, 3001, 2000)
    ws.fill_(-1)
    off = torch.full((3,), -1, dtype=torch.int64, device=DEV)
    enc.plan(d, ws, off)
    total = int(off[-1].item())
    out = torch.full((total,), 0xFF, dtype=torch.uint8, device=DEV)
    enc.write(d, ws, off, out)
    o = off.cpu().numpy()
    host = out.cpu().numpy()
    assert [host[o[i]:o[i + 1]].tobytes() for i in range(2)] == whole[3:5]


def test_graph_replay_equals_eager(emul):  # noqa: F811
    rng = np.random.default_rng(5)
    b, n = 3, 2000
    v = torch.from_numpy(_meshes(rng, b, n, edge=False)).to(DEV)
    tri = rng.integers(1, n + 1, (3, 1500))
    col = rng.integers(0, 256, (n, 3)).astype(np.uint8)
    t = ObjTables(tri, n, col, None, b)
    enc = obj_encoder(DEV)
    d = t.desc(v, 0, DEV)
    ws = enc.workspace(b, n, 1500)
    off = torch.empty(b + 1, dtype=torch.int64, device=DEV)
    out = torch.empty(int(2.5 * b * (n * 60 + 1500 * 20)), dtype=torch.uint8, device=DEV)
    enc.plan(d, ws, off)
    enc.write(d, ws, off, out)                                                              # eager first
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        enc.plan(d, ws, off)
        enc.write(d, ws, off, out)
    for rep in range(3):
        with np.errstate(invalid='ignore'):                                                # signalling NaNs among the edges
            v.copy_(torch.from_numpy(_meshes(rng, b, n, edge=rep == 0) * np.float32(10.0 ** rep)).to(DEV))
        out.fill_(0xFF)
        g.replay()
        torch.cuda.synchronize()
        o = off.cpu().numpy()
        host = out.cpu().numpy()
        replayed = [host[o[i]:o[i + 1]].tobytes() for i in range(b)]
        assert replayed == t.encode(v), rep
        assert replayed == [emul_file(emul, v[i].cpu().numpy(), tri, col) for i in range(b)], rep


def test_refusals_launch_nothing(synth_pack):
    model = _checkpoint('mobilenet_v2')
    frames = np.stack([synthetic.make_scene_u8(240, 320, i) for i in range(2)])
    rects = [[[10.0, 10.0, 150.0, 170.0, 0.9]], [[40.0, 30.0, 200.0, 220.0, 0.8]]]
    model.obj_batch(frames, rects=rects)
    eng = model._engine(model._compute_device())
    enc = obj_encoder(DEV)
    v = torch.from_numpy(_meshes(np.random.default_rng(6), 2, 100)).to(DEV)
    tri = np.array([[1], [2], [3]])
    t = ObjTables(tri, 100)
    ws = enc.workspace(2, 100, 1)
    off = torch.full((3,), -7, dtype=torch.int64, device=DEV)     # a launched plan would write offsets (0 first)
    out = torch.full((8000,), 0xAB, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    before = (eng.launch_count, enc.launches)
    lib = _lib.load()
    st = torch.cuda.current_stream(DEV).cuda_stream
    bad = np.array([0, 100], np.int32)
    keep_dev = torch.from_numpy(bad).to(DEV)
    for field, value in (('tri_order', 2), ('stride_vertex', 0), ('batch', 0), ('keep', None)):
        e = t.desc(v, 0, DEV)
        if field == 'keep':
            e.keep_host, e.keep_dev, e.n_keep = bad.ctypes.data, keep_dev.data_ptr(), 2
        else:
            setattr(e, field, value)
        assert lib.syn_obj_plan(C.byref(e), ws.data_ptr(), ws.numel() * 8, off.data_ptr(), st) == 1, field
        assert lib.syn_obj_write(C.byref(e), ws.data_ptr(), ws.numel() * 8, off.data_ptr(), out.data_ptr(), out.numel(), st) == 1
    for call in (lambda: obj_bytes(v, tri, keep=[0, 100]), lambda: obj_bytes(v.double(), tri),
                 lambda: obj_bytes(v, tri, np.full((100, 3), 0.5))):
        with pytest.raises((ValueError, TypeError)):
            call()
    torch.cuda.synchronize()
    # the OBJ entries are handle-free and ObjEncoder.launches counts only its own calls: the counters show that the Python
    # refusals reached neither; the untouched offsets and output show that the raw C refusals launched nothing
    assert (eng.launch_count, enc.launches) == before
    assert bool((out == 0xAB).all()) and bool((off == -7).all())


# ---- the models -------------------------------------------------------------------------------------------------------------
def _checkpoint(arch):
    if arch == 'mobilenet_v2':
        return make_model(synth_model.build_state_dict(0))
    if arch.startswith('resnet'):
        return make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
    return make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)


def _loop(outputs, tri, colors=None, keep=None):
    """The reference's write_obj (or write_obj_with_colors on the kept vertices) per face, restated in Python: the text
    the device must reproduce, from a source independent of its kernels."""
    return [python_obj(mesh if keep is None else mesh[:, keep], tri, colors) for mesh in outputs[1]]


RECTS = [[[10.0, 20.0, 200.0, 240.0, 0.9], [150.0, 100.0, 330.0, 300.0, 0.8]], [], [[-30.0, 40.0, 120.0, 200.0, 0.7]],
         [[500.0, 300.0, 800.0, 620.0, 0.9]]]


@pytest.mark.parametrize('arch', ['mobilenet_v2', 'resnet18', 'mobilenet_05'])
def test_obj_images_and_batch_equal_the_per_face_loop(synth_pack, arch):
    model = _checkpoint(arch)
    tri = model.triangles.cpu().numpy() + 1
    sizes = [(360, 480), (1, 1), (250, 333), (720, 1080)]
    images = [synthetic.make_scene_u8(h, w, 7 * i) for i, (h, w) in enumerate(sizes)]
    outputs = model.get_all_outputs_images(images, rects=RECTS)
    got = model.obj_images(images, rects=RECTS)
    assert [len(g) for g in got] == [2, 0, 1, 1]
    for i in range(4):
        assert got[i] == _loop(outputs[i], tri), f'{arch} image {i}'
    model.dense_chunk_bytes = 3 * 4 * 53215 * 2 + 1                                     # two faces per chunk
    try:
        assert model.obj_images([torch.from_numpy(im).to(DEV) for im in images], rects=RECTS) == got
    finally:
        del model.dense_chunk_bytes
    frames = np.stack([synthetic.make_scene_u8(720, 1080, 50 + i) for i in range(4)])
    outs = model.get_all_outputs_batch(frames, rects=RECTS)
    assert model.obj_batch(frames, rects=RECTS) == [_loop(outs[i], tri) for i in range(4)]


def test_obj_with_kept_vertices_and_colours(synth_pack):
    model = _checkpoint('mobilenet_v2')
    rng = np.random.default_rng(8)
    frames = np.stack([synthetic.make_scene_u8(480, 640, 30 + i) for i in range(2)])
    rects = [[[100.0, 80.0, 300.0, 300.0, 0.9]], [[50.0, 50.0, 250.0, 280.0, 0.9], [300.0, 100.0, 500.0, 330.0, 0.7]]]
    outs = model.get_all_outputs_batch(frames, rects=rects)
    nver = outs[0][1][0].shape[1]
    keep = np.sort(rng.choice(nver, 40000, replace=False))
    tri_del = rng.integers(1, 40001, (3, 70000)).astype(np.int32)
    colors = rng.integers(0, 256, (40000, 3)).astype(np.uint8).astype(np.float32)
    got = model.obj_batch(frames, rects=rects, keep=keep, colors=colors, triangles=tri_del)
    assert got == [_loop(outs[i], tri_del, colors, keep) for i in range(2)]
    plain = model.obj_batch(frames, rects=rects, keep=keep, triangles=tri_del)
    assert plain == [_loop(outs[i], tri_del, None, keep) for i in range(2)]


def test_more_meshes_than_one_call_takes():
    """70 000 one-vertex meshes: chunked at the 65 535 meshes one syn_obj_plan call accepts."""
    v = torch.zeros((70000, 3, 1), dtype=torch.float32, device=DEV)
    v[-1, 0, 0] = 1.5
    got = obj_bytes(v, np.zeros((3, 0), np.int64))
    assert len(got) == 70000 and got[0] == b'v 0.0000 0.0000 0.0000\n' and got[-1] == b'v 1.5000 0.0000 0.0000\n'


def test_threads_on_their_own_streams_share_the_encoder_and_a_model(synth_pack):
    """Two host threads, each on its own CUDA stream, encode at once through one model and the one encoder of the device:
    meshes of different sizes with obj_bytes, and obj_images.  Every result equals the single-threaded bytes."""
    from test_gpu_concurrency import ITERS, run_threads
    model = _checkpoint('mobilenet_v2')
    rng = np.random.default_rng(10)
    meshes = [torch.from_numpy(_meshes(rng, 3, 900)).to(DEV), torch.from_numpy(_meshes(rng, 6, 20000)).to(DEV)]
    tris = [rng.integers(1, 900, (3, 1200)), rng.integers(1, 20000, (3, 30000))]
    images = [[synthetic.make_scene_u8(240, 320, 60)], [synthetic.make_scene_u8(480, 640, 61), synthetic.make_scene_u8(300, 400, 62)]]
    rects = [[[[20.0, 20.0, 180.0, 200.0, 0.9]]], [[[50.0, 40.0, 260.0, 290.0, 0.9], [300.0, 100.0, 520.0, 360.0, 0.8]],
                                                   [[10.0, 10.0, 200.0, 230.0, 0.7]]]]

    def work(t, i):
        if i % 2:
            return model.obj_images(images[t], rects=rects[t])
        return obj_bytes(meshes[t], tris[t])

    want = [[work(t, i) for i in range(2)] for t in range(2)]
    torch.cuda.synchronize()
    got = run_threads(work)
    for t in range(2):
        for i in range(ITERS):
            assert got[t][i] == want[t][i % 2], f'thread {t} iteration {i}'
