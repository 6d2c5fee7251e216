"""The UV texture path on the H100: syn_uv_sample against the host restatement of its gather (which test_uv_host.py holds
to numpy's flip-and-index), syn_mesh_lighting_textures against the shared-texture lighting, the reference's own textured
OBJ files and overlays (the committed golden digests), and the models' uv_obj_* / uv_overlay_* against
get_all_outputs_* followed by the per-face loop of artistic.py and uv_texture_realFaces.py.  Every equality is bit for
bit."""
import ctypes as C
import hashlib
import json

import cv2
import numpy as np
import pytest
import torch

from golden.make_golden_uv import OUT_JSON, colors_uv, golden_inputs
from oracle import synth_mbv1, synth_model, synth_resnet
from oracle.stage_check import make_model
from synergynet_b200 import Sim3DR, _lib, synthetic
from synergynet_b200.inference import RENDER_CFG, ObjTables, UVLayout, UVMaps, pack_images, square_roi, uv_maps_host
from test_gpu_render_images import FILLS, poisoned_empty
from test_obj_emulation import python_obj
from test_uv_host import sample_host

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
CFG = Sim3DR._light_cfg(**RENDER_CFG)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---- syn_uv_sample ------------------------------------------------------------------------------------------------------
def _ragged(seed):
    uv, keep, tri = synthetic.make_uv_layout(seed, nver=7000)
    layout = UVLayout(uv, keep, tri)
    maps = [synthetic.make_uv_map(h, w, seed=seed + i) for i, (h, w) in enumerate([(256, 256), (300, 512), (512, 300), (257, 999)])]
    return layout, maps


def test_uv_sample_equals_the_emulation_on_ragged_maps():
    layout, maps = _ragged(1)
    face_map = [3, 0, 0, 2, 1, 1, 3, 2, 0]
    uvm = UVMaps(layout, maps, face_map, DEV)
    want_t, want_c = sample_host(layout, maps, face_map)
    for a, b in ((0, 9), (0, 1), (2, 7), (8, 9)):
        t, c = uvm.sample(a, b, texture=True, colors=True)
        assert t.cpu().numpy().tobytes() == want_t[a:b].tobytes() and np.array_equal(c.cpu().numpy(), want_c[a:b]), (a, b)
        t1, c1 = uvm.sample(a, b)
        assert c1 is None and torch.equal(t1, t)
        t2, c2 = uvm.sample(a, b, texture=False, colors=True)
        assert t2 is None and torch.equal(c2, c)


def test_uv_sample_stale_poisoned_and_graph_replay():
    layout, maps = _ragged(2)
    face_map = [1, 2, 3, 0, 2]
    uvm = UVMaps(layout, maps, face_map, DEV)
    want_t, want_c = sample_host(layout, maps, face_map)
    for byte in (None,) + tuple(FILLS):
        if byte is None:
            t, c = uvm.sample(0, 5, colors=True)
        else:
            with poisoned_empty(byte, byte):
                t, c = uvm.sample(0, 5, colors=True)
        torch.cuda.synchronize()
        assert t.cpu().numpy().tobytes() == want_t.tobytes() and np.array_equal(c.cpu().numpy(), want_c), byte
    # one graph: the sampler, then the per-mesh lighting of its texture; replays follow new map bytes and new meshes
    n = layout.n_keep
    r = Sim3DR.MeshRenderer(layout.render_tri, n, DEV)
    verts = torch.from_numpy(synthetic.make_render_meshes(5, 200, 200, seed=3, rows=70, cols=100)[:, :, layout.keep]).to(DEV)
    v = verts.transpose(1, 2)
    nrm = r.normals(v)
    tex = torch.empty((5, n, 3), dtype=torch.float32, device=DEV)
    col = torch.empty((5, n, 3), dtype=torch.int64, device=DEV)
    stats = torch.empty((5, 6), dtype=torch.int32, device=DEV)
    lit = torch.empty((5, n, 3), dtype=torch.float32, device=DEV)
    pa, pb, pc = uvm._parts
    fm = np.ascontiguousarray(uvm.face_map)
    lib = _lib.load()

    def calls():
        st = torch.cuda.current_stream(DEV).cuda_stream
        _lib.check(lib.syn_uv_sample(uvm.dev[pc:].data_ptr(), uvm.map_bytes, uvm.table.ctypes.data, uvm.dev.data_ptr(), uvm.n_maps,
                                     uvm.texels.ctypes.data, uvm.dev[pa:].data_ptr(), n, fm.ctypes.data, uvm.dev[pb:].data_ptr(), 5,
                                     tex.data_ptr(), col.data_ptr(), st))
        sv = [int(s) for s in v.stride()]
        _lib.check(lib.syn_mesh_lighting_textures(v.data_ptr(), sv[0], sv[1], sv[2], 5, n, nrm.data_ptr(), C.byref(CFG), tex.data_ptr(),
                                                  3 * n, stats.data_ptr(), lit.data_ptr(), st))

    calls()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        calls()
    for rep in range(2):
        new_maps = [synthetic.make_uv_map(m.shape[0], m.shape[1], seed=90 + rep + i) for i, m in enumerate(maps)]
        uvm.dev[pc:].view(torch.uint8)[:uvm.map_bytes].copy_(torch.from_numpy(np.concatenate([m.reshape(-1) for m in new_maps])))
        verts.mul_(1.01)
        tex.fill_(-1.0), col.fill_(-1), lit.fill_(-1.0)
        g.replay()
        torch.cuda.synchronize()
        want_t, want_c = sample_host(layout, new_maps, face_map)
        assert tex.cpu().numpy().tobytes() == want_t.tobytes() and np.array_equal(col.cpu().numpy(), want_c), rep
        want = r.colors(v, nrm, CFG, torch.from_numpy(want_t).to(DEV))     # NaN at the kept vertices no triangle touches
        assert torch.equal(lit.view(torch.int32), want.view(torch.int32)), rep


# ---- syn_mesh_lighting_textures --------------------------------------------------------------------------------------------
def test_lighting_with_a_texture_per_mesh():
    tri = synthetic.make_render_topology(40, 50)
    r = Sim3DR.MeshRenderer(tri, 2000, DEV)
    v = torch.from_numpy(synthetic.make_render_meshes(4, 120, 160, seed=5, rows=40, cols=50)).to(DEV).transpose(1, 2)
    nrm = r.normals(v)
    rng = np.random.default_rng(6)
    tex = torch.from_numpy(rng.integers(0, 256, (4, 2000, 3)).astype(np.float32) / np.float32(255)).to(DEV)
    got = r.colors(v, nrm, CFG, tex)
    for b in range(4):
        assert torch.equal(got[b], r.colors(v[b:b + 1], nrm[b:b + 1], CFG, tex[b])[0]), b
    # stride 0 is the shared texture: the bits of syn_mesh_lighting
    lib = _lib.load()
    st = torch.cuda.current_stream(DEV).cuda_stream
    stats = torch.empty((4, 6), dtype=torch.int32, device=DEV)
    out = torch.full((4, 2000, 3), float('nan'), device=DEV)
    sv = [int(s) for s in v.stride()]
    _lib.check(lib.syn_mesh_lighting_textures(v.data_ptr(), sv[0], sv[1], sv[2], 4, 2000, nrm.data_ptr(), C.byref(CFG), tex[2].data_ptr(),
                                              0, stats.data_ptr(), out.data_ptr(), st))
    assert torch.equal(out, r.colors(v, nrm, CFG, tex[2]))
    with pytest.raises(ValueError, match=r'\(B, nver, 3\)'):
        r.colors(v, nrm, CFG, tex[:3])


# ---- the reference's files and overlays (golden digests) -----------------------------------------------------------------------
def test_golden_obj_and_overlays():
    doc = json.load(open(OUT_JSON))
    for k, case in enumerate(doc['cases']):
        uv, keep, tri, uv_map, image, meshes = golden_inputs(k)
        assert [_sha(a) for a in (uv, keep, tri, uv_map, image, meshes)] == case['inputs'], f'case {k}: inputs drifted'
        layout = UVLayout(uv, keep, tri)
        maps = uv_maps_host(uv_map, 1, False)
        f = meshes.shape[0]
        uvm = UVMaps(layout, maps, [0] * f, DEV)
        tex, col = uvm.sample(0, f, colors=True)
        v = torch.from_numpy(meshes).to(DEV)
        texts = ObjTables(tri, meshes.shape[2], None, keep, f).encode(v, 0, colors_dev=col)
        got = [{'bytes': len(t), 'sha256': hashlib.sha256(t).hexdigest()} for t in texts]
        assert got == case['obj'], f'case {k}: OBJ files'
        assert texts[0] == python_obj(meshes[0][:, keep], tri, colors_uv(uv, keep, uv_map).astype(np.float32))
        if case['overlay'] is None:
            continue
        r = Sim3DR.MeshRenderer(layout.render_tri, layout.n_keep, DEV)
        kv = v[:, :, torch.from_numpy(keep).to(DEV)].transpose(1, 2)
        blended, solid = r.render_images(pack_images([image], DEV), kv, [f], CFG, tex, 0.6)
        assert _sha(solid.data.cpu().numpy()) == case['overlay']['solid'], f'case {k}: solid overlay'
        assert _sha(blended.data.cpu().numpy()) == case['overlay']['blended'], f'case {k}: blended'


# ---- the models ---------------------------------------------------------------------------------------------------------------
def _checkpoint(arch):
    if arch == 'mobilenet_v2':
        m = make_model(synth_model.build_state_dict(0))
    elif arch.startswith('resnet'):
        m = make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
    else:
        m = make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)
    m.resize_interpolation = 'linear'                       # artistic.py:95, uv_texture_realFaces.py:88
    return m


@pytest.fixture(scope='module')
def layout(synth_pack):
    return UVLayout(*synthetic.make_uv_layout(0))


def _maps(n, seed=0):
    return [synthetic.make_uv_map(*hw, seed=seed + i) for i, hw in zip(range(n), [(256, 256), (300, 512), (512, 300), (256, 257)] * 4)]


def _obj_loop(layout, outputs, maps):
    """artistic.py's writer per face, restated: write_obj_with_colors(m[:, keep], deletedTri, colors_uv[keep] as float32)."""
    out = []
    for i, (_, meshes, _) in enumerate(outputs):
        col = np.flip(maps[i], 0)[layout.coord_u, layout.coord_v][layout.keep, :3].astype(np.float32)
        out.append([python_obj(m[:, layout.keep], layout.deleted_tri, col) for m in meshes])
    return out


def _overlay_loop(layout, images, outputs, maps, alpha=0.6):
    """uv_texture_realFaces.py's overlay per image: a RenderPipeline call per face with a fresh texture, then the blend."""
    app = Sim3DR.RenderPipeline(**RENDER_CFG)
    want = []
    for i, (im, (_, meshes, _)) in enumerate(zip(images, outputs)):
        overlap = im.copy()
        for m in meshes:
            tex = np.flip(maps[i], 0)[layout.coord_u, layout.coord_v][layout.keep].astype(np.float32) / 255.0
            overlap = app(np.ascontiguousarray(m[:, layout.keep].T), layout.render_tri, overlap, texture=tex)
        want.append((cv2.addWeighted(im, 1 - alpha, overlap, alpha, 0), overlap))
    return want


def _same(got, want, where):
    blended, solid = got
    assert len(blended) == len(solid) == len(want), where
    for i, (wb, ws) in enumerate(want):
        gs = solid[i].cpu().numpy() if isinstance(solid[i], torch.Tensor) else solid[i]
        gb = blended[i].cpu().numpy() if isinstance(blended[i], torch.Tensor) else blended[i]
        assert np.array_equal(gs, ws), f'{where}: solid overlay of image {i}'
        assert np.array_equal(gb, wb), f'{where}: blended image {i}'


SIZES = [(360, 480), (1, 1), (250, 333), (720, 1080)]
RECTS = [[[10.0, 20.0, 200.0, 240.0, 0.9], [150.0, 100.0, 330.0, 300.0, 0.8]], [], [[-30.0, 40.0, 120.0, 200.0, 0.7]],
         [[900.0, 300.0, 1200.0, 620.0, 0.9]]]


@pytest.mark.parametrize('arch', ['mobilenet_v2', 'resnet18', 'mobilenet_05'])
def test_uv_images_and_batch_equal_the_per_face_loop(layout, arch):
    model = _checkpoint(arch)
    images = [synthetic.make_scene_u8(h, w, 7 * i) for i, (h, w) in enumerate(SIZES)]
    maps = _maps(4)
    outputs = model.get_all_outputs_images(images, rects=RECTS)
    objs = model.uv_obj_images(images, maps, layout, rects=RECTS)
    assert [len(o) for o in objs] == [2, 0, 1, 1]
    assert objs == _obj_loop(layout, outputs, maps), arch
    want = _overlay_loop(layout, images, outputs, maps)
    _same(model.uv_overlay_images(images, maps, layout, rects=RECTS), want, f'{arch} uv_overlay_images')
    model.dense_chunk_bytes = 3 * 4 * 53215 * 2 + 1                                     # two faces per chunk
    try:
        dev_images = [torch.from_numpy(im).to(DEV) for im in images]
        _same(model.uv_overlay_images(dev_images, maps, layout, rects=RECTS), want, f'{arch} CUDA images, chunks')
        assert model.uv_obj_images(dev_images, maps, layout, rects=RECTS) == objs
    finally:
        del model.dense_chunk_bytes
    frames = np.stack([synthetic.make_scene_u8(720, 1080, 50 + i) for i in range(4)])
    outs = model.get_all_outputs_batch(frames, rects=RECTS)
    assert model.uv_obj_batch(frames, maps, layout, rects=RECTS) == _obj_loop(layout, outs, maps)
    got = model.uv_overlay_batch(frames, maps, layout, rects=RECTS)
    want = _overlay_loop(layout, list(frames), outs, maps)
    _same((list(got[0]), list(got[1])), want, f'{arch} uv_overlay_batch')
    # one map for every frame
    shared = [maps[2]] * 4
    assert model.uv_obj_batch(frames, maps[2], layout, rects=RECTS) == _obj_loop(layout, outs, shared)


def test_rois_as_given_equal_the_realfaces_chain(layout):
    """uv_texture_realFaces.py crops [0, 0, 256, 256, 1.0] as given; a detector box whose square_roi is that ROI gives the
    same crop through get_all_outputs, so that chain is the reference here."""
    model = _checkpoint('mobilenet_v2')
    roi = [0, 0, 256, 256, 1.0]
    rect = [21.2, 21.2, 234.8, 234.8, 1.0]
    assert square_roi(rect) == roi
    images = [synthetic.make_scene_u8(256, 256, 70 + i) for i in range(3)]
    maps = _maps(3, seed=5)
    outputs = [model.get_all_outputs(im, rects=[rect]) for im in images]
    objs = model.uv_obj_images(images, maps, layout, rois=[roi])
    assert objs == _obj_loop(layout, outputs, maps)
    assert model.uv_obj_images(images, maps, layout, rois=[[roi]] * 3) == objs
    assert model.uv_obj_batch(np.stack(images), maps, layout, rois=[roi]) == objs
    want = _overlay_loop(layout, images, outputs, maps)
    _same(model.uv_overlay_images(images, maps, layout, rois=[roi]), want, 'rois')
    # one face: utils/render.render(img, [m[:, keep]], tex=tex, connectivity=deletedTri - 1) itself
    for i in range(3):
        m = outputs[i][1][0]
        tex = np.flip(maps[i], 0)[layout.coord_u, layout.coord_v][layout.keep].astype(np.float32) / 255.0
        res, overlap = Sim3DR.render(images[i], [m[:, layout.keep]], layout.render_tri, alpha=0.6, tex=tex, cfg=RENDER_CFG)
        assert np.array_equal(overlap, want[i][1]) and np.array_equal(res, want[i][0])


def test_stale_and_poisoned_outputs(layout):
    model = _checkpoint('mobilenet_v2')
    images = [synthetic.make_scene_u8(h, w, 3 * i) for i, (h, w) in enumerate([(300, 400), (200, 256)])]
    rects = [[[40.0, 30.0, 250.0, 260.0, 0.9], [200.0, 20.0, 390.0, 240.0, 0.8]], [[20.0, 20.0, 180.0, 190.0, 0.9]]]
    maps = _maps(2, seed=9)
    cases = {'overlay': lambda: model.uv_overlay_images(images, maps, layout, rects=rects),
             'obj': lambda: model.uv_obj_images(images, maps, layout, rects=rects)}
    clean = {k: fn() for k, fn in cases.items()}
    eng = model._engine(model._compute_device())
    for byte in FILLS:
        eng.debug_fill_workspaces(byte)
        with poisoned_empty(byte, byte):
            got = {k: fn() for k, fn in cases.items()}
        torch.cuda.synchronize()
        assert got['obj'] == clean['obj'], byte
        _same(got['overlay'], list(zip(*clean['overlay'])), f'fill 0x{byte:02X}')


def test_refusals_launch_nothing(layout):
    model = _checkpoint('mobilenet_v2')
    images = [synthetic.make_scene_u8(200, 300, 1)]
    rects = [[[40.0, 30.0, 180.0, 190.0, 0.9]]]
    m = _maps(1)[0]
    model.uv_overlay_images(images, m, layout, rects=rects)
    eng = model._engine(model._compute_device())
    r = Sim3DR._renderer_for(layout.render_tri, layout.n_keep)
    torch.cuda.synchronize()
    before = (eng.launch_count, r.launches)
    for kw in ({'uv_maps': m[:, :, :1]}, {'uv_maps': m.astype(np.uint16)}, {'uv_maps': synthetic.make_uv_map(256, 256, channels=4)},
               {'uv_maps': m[:200]}, {'rois': rects}, {'rects': None}):
        args = {'uv_maps': m, 'rects': rects, **kw}
        with pytest.raises((ValueError, IndexError)):
            model.uv_overlay_images(images, args['uv_maps'], layout, rects=args['rects'], rois=args.get('rois'))
    uvm = UVMaps(layout, [m], [0], DEV)
    lib = _lib.load()
    out = torch.full((1, layout.n_keep, 3), 7.0, device=DEV)
    bad = np.ascontiguousarray(uvm.texels.copy())
    bad[0, -1] = (256, 0)
    pa, pb, pc = uvm._parts
    fm = np.zeros(1, np.int32)
    st = torch.cuda.current_stream(DEV).cuda_stream
    assert lib.syn_uv_sample(uvm.dev[pc:].data_ptr(), uvm.map_bytes, uvm.table.ctypes.data, uvm.dev.data_ptr(), 1, bad.ctypes.data,
                             uvm.dev[pa:].data_ptr(), layout.n_keep, fm.ctypes.data, uvm.dev[pb:].data_ptr(), 1, out.data_ptr(), None,
                             st) == 4
    torch.cuda.synchronize()
    assert (eng.launch_count, r.launches, uvm.launches) == before + (0,)
    assert bool((out == 7.0).all())


def test_threads_on_their_own_streams_share_a_model(layout):
    from test_gpu_concurrency import ITERS, run_threads
    model = _checkpoint('mobilenet_v2')
    images = [[synthetic.make_scene_u8(240, 320, 60)], [synthetic.make_scene_u8(480, 640, 61), synthetic.make_scene_u8(300, 400, 62)]]
    rects = [[[[20.0, 20.0, 180.0, 200.0, 0.9]]], [[[50.0, 40.0, 260.0, 290.0, 0.9], [300.0, 100.0, 520.0, 360.0, 0.8]],
                                                   [[10.0, 10.0, 200.0, 230.0, 0.7]]]]
    maps = [_maps(1, 20), _maps(2, 30)]

    def work(t, i):
        if i % 2:
            return model.uv_obj_images(images[t], maps[t], layout, rects=rects[t])
        b, s = model.uv_overlay_images(images[t], maps[t], layout, rects=rects[t])
        return [x.copy() for x in b + s]

    want = [[work(t, i) for i in range(2)] for t in range(2)]
    torch.cuda.synchronize()
    got = run_threads(work)
    for t in range(2):
        for i in range(ITERS):
            w, g = want[t][i % 2], got[t][i]
            assert len(w) == len(g) and all((a == b) if isinstance(a, list) else np.array_equal(a, b) for a, b in zip(w, g)), (t, i)
