"""Parity of the Sim3DR and FaceBoxes post-processing kernels (SURVEY.md section 8 rows f2, f3) on the H100, through the
C ABI: bit-exact against the C oracle and the golden vectors recorded from the reference for normals, rasterisation and
NMS index lists; lighting and box decode to the tolerance their one non-reproducible library call (pow / exp) allows."""
import os

import numpy as np
import pytest
import torch

from oracle import render_port as rp
from synergynet_b200 import Sim3DR, _lib, detect, synthetic
from synergynet_b200.inference import RENDER_CFG

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'render_vectors.npz')
LIGHT_TOL = 2e-7


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLD, allow_pickle=False))


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda', 0)


def test_native_library_is_the_one_running():
    lib = _lib.load()
    assert lib.syn_abi_version() == 1 and hasattr(lib, 'syn_rasterize') and hasattr(lib, 'syn_nms')


def test_normals_bit_exact_both_layouts(gold, dev):
    tri, verts = gold['render_tri'], gold['render_verts']
    r = Sim3DR.MeshRenderer(tri, verts.shape[2], dev)
    planes = torch.from_numpy(verts).to(dev)                                   # (B,3,N) like the dense 3DMM output
    n1 = r.normals(planes.transpose(1, 2))                                     # strided view
    n2 = r.normals(planes.transpose(1, 2).contiguous())                        # (B,N,3) like the reference's arrays
    assert torch.equal(n1, n2)
    assert np.array_equal(n1.cpu().numpy(), gold['render_normals'])


def test_lighting(gold, dev):
    tri, verts = gold['render_tri'], gold['render_verts']
    r = Sim3DR.MeshRenderer(tri, verts.shape[2], dev)
    v = torch.from_numpy(verts).to(dev).transpose(1, 2)
    nrm = torch.from_numpy(gold['render_normals']).to(dev)
    light = r.colors(v, nrm, Sim3DR._light_cfg(**RENDER_CFG)).cpu().numpy()
    assert np.abs(light - gold['render_light']).max() <= LIGHT_TOL
    tex = torch.rand((verts.shape[2], 3), generator=torch.Generator().manual_seed(0))
    lt = r.colors(v, nrm, Sim3DR._light_cfg(**RENDER_CFG), tex).cpu().numpy()
    assert np.array_equal(lt, tex.numpy()[None] * light)


def test_rasterize_bit_exact_vs_reference_vectors(gold, dev):
    tri, verts, bg = gold['render_tri'], gold['render_verts'], gold['render_bg']
    r = Sim3DR.MeshRenderer(tri, verts.shape[2], dev)
    v = torch.from_numpy(verts).to(dev).transpose(1, 2)
    colors = torch.from_numpy(gold['render_light']).to(dev)
    # the batch drawn in one call = the reference after its third sequential mesh; prefixes = its intermediate images
    for nb in (1, 2, 3):
        img = torch.from_numpy(bg.copy()).to(dev)
        _, depth = r.rasterize(img, v[:nb], colors[:nb], return_depth=True)
        assert np.array_equal(img.cpu().numpy(), gold['render_steps'][nb - 1])
        for k in range(nb):
            _, d = rp.rasterize(np.ascontiguousarray(verts[k].T), tri, gold['render_light'][k], bg.copy(), return_depth=True)
            assert np.array_equal(depth[k].cpu().numpy(), d)
    for key, rev in (('raster_plain', False), ('raster_reverse', True)):
        img = torch.from_numpy(bg.copy()).to(dev)
        r.rasterize(img, v[:1], torch.from_numpy(gold['raster_colors']).to(dev)[None], reverse=rev)
        assert np.array_equal(img.cpu().numpy(), gold[key])


def test_rasterize_ties_large_and_degenerate_triangles(dev):
    ver = np.array([[-30, -20, 1], [90, -10, 1], [20, 100, 1], [5, 5, 1], [40, 8, 1], [12, 50, 1], [200, 200, 5], [210, 200, 5],
                    [200, 210, 5], [10, 10, 3], [10, 10, 3], [30, 30, 3]], np.float32)
    tri = np.array([[0, 1, 2], [3, 4, 5], [0, 1, 2], [6, 7, 8], [9, 10, 11], [5, 4, 3]], np.int32)
    col = np.random.default_rng(0).uniform(0, 1, (12, 3)).astype(np.float32)
    bg = np.full((48, 64, 3), 17, np.uint8)
    want, dwant = rp.rasterize(ver, tri, col, bg.copy(), return_depth=True)
    r = Sim3DR.MeshRenderer(tri, 12, dev)
    img = torch.from_numpy(bg.copy()).to(dev)
    _, depth = r.rasterize(img, torch.from_numpy(ver).to(dev)[None], torch.from_numpy(col).to(dev)[None], return_depth=True)
    assert np.array_equal(img.cpu().numpy(), want) and np.array_equal(depth[0].cpu().numpy(), dwant)


def test_rasterize_signed_zero_depth_tie(dev):
    """Coplanar copies of one triangle at depth -0 and then +0 tie in the reference's serial `>`: the first one stays."""
    xy = [[2, 2], [30, 3], [6, 25]]
    ver = np.array([p + [-0.0] for p in xy] + [p + [0.0] for p in xy], np.float32)
    tri = np.array([[0, 1, 2], [3, 4, 5]], np.int32)
    col = np.array([[0.9, 0.1, 0.1]] * 3 + [[0.1, 0.1, 0.9]] * 3, np.float32)
    bg = np.zeros((32, 32, 3), np.uint8)
    want, dwant = rp.rasterize(ver, tri, col, bg.copy(), return_depth=True)
    r = Sim3DR.MeshRenderer(tri, 6, dev)
    img = torch.from_numpy(bg.copy()).to(dev)
    _, depth = r.rasterize(img, torch.from_numpy(ver).to(dev)[None], torch.from_numpy(col).to(dev)[None], return_depth=True)
    assert (want[..., 0] == 229).any() and np.array_equal(img.cpu().numpy(), want)
    assert np.array_equal(depth[0].cpu().numpy(), dwant)


def test_pipeline_reference_shaped_api(gold):
    """The numpy-in / numpy-out functions with the reference's names and call signatures (Sim3DR/Sim3DR.py, lighting.py)."""
    tri, verts, bg = gold['render_tri'], gold['render_verts'], gold['render_bg']
    ver0 = np.ascontiguousarray(verts[0].T)
    assert np.array_equal(Sim3DR.get_normal(ver0, tri), gold['render_normals'][0])
    canvas = bg.copy()
    out = Sim3DR.rasterize(ver0, tri, gold['raster_colors'], bg=canvas)
    assert out is canvas and np.array_equal(out, gold['raster_plain'])
    assert np.array_equal(Sim3DR.rasterize(ver0, tri, gold['raster_colors'], bg=bg.copy(), reverse=True), gold['raster_reverse'])
    app = Sim3DR.RenderPipeline(**RENDER_CFG)
    overlap = bg.copy()
    for b in range(3):                                                      # utils/render.py:40-45
        overlap = app(np.ascontiguousarray(verts[b].T), tri, overlap)
        diff = np.abs(overlap.astype(np.int32) - gold['render_steps'][b].astype(np.int32))
        assert diff.max() <= 1 and (diff != 0).mean() < 1e-3               # light is 1 ulp from numpy's at a few vertices
    tex = np.ones_like(ver0)
    app(ver0, tri, bg.copy(), texture=tex)                                   # `texture *= light` happens in place
    assert np.abs(tex - gold['render_light'][0]).max() <= LIGHT_TOL
    with pytest.raises(ValueError):
        Sim3DR.rasterize(ver0, tri, gold['raster_colors'], bg=bg.astype(np.float32))


def test_full_size_batch_against_the_oracle(dev):
    """53 215 vertices / 105 408 triangles per mesh, four meshes on a 720 x 1080 canvas, read in place from a (B,3,N) tensor."""
    tri = synthetic.make_render_topology()
    verts = synthetic.make_render_meshes(4, 720, 1080, seed=0)
    bg = np.random.default_rng(1).integers(0, 256, (720, 1080, 3), dtype=np.uint8)
    r = Sim3DR.MeshRenderer(tri, verts.shape[2], dev)
    v = torch.from_numpy(verts).to(dev).transpose(1, 2)
    nrm = r.normals(v)
    want_n = np.stack([rp.get_normal(np.ascontiguousarray(verts[b].T), tri) for b in range(4)])
    assert np.array_equal(nrm.cpu().numpy(), want_n)
    col = r.colors(v, nrm, Sim3DR._light_cfg(**RENDER_CFG))
    want_c = np.stack([rp.lighting(np.ascontiguousarray(verts[b].T), want_n[b]) for b in range(4)])
    assert np.abs(col.cpu().numpy() - want_c).max() <= LIGHT_TOL
    img = torch.from_numpy(bg.copy()).to(dev)
    r.rasterize(img, v, col)
    want = bg.copy()
    col_host = col.cpu().numpy()
    for b in range(4):                                                      # same colours in: the uint8 image must be identical
        want = rp.rasterize(np.ascontiguousarray(verts[b].T), tri, col_host[b], want)
    assert np.array_equal(img.cpu().numpy(), want)
    assert (want != bg).any(axis=2).sum() > 50000
    blended, overlap = Sim3DR.render(bg, list(verts), tri)
    assert np.array_equal(overlap, want) and blended.shape == bg.shape


# ---- FaceBoxes post-processing --------------------------------------------------------------------------------------------
def _nms_dev(dets_sorted, thr, mode, dev):
    keep, n = detect.nms_device(torch.from_numpy(np.ascontiguousarray(dets_sorted)).to(dev), thr, mode)
    return keep[:int(n.item())].cpu().numpy()


def test_nms_index_lists_bit_exact(gold, dev):
    d = gold['nms_dets']
    for thr, key in ((0.3, 'nms_keep_3'), (0.5, 'nms_keep_5')):
        assert detect.py_cpu_nms(d, thr) == gold[key].tolist()
        assert detect.cpu_nms(d, thr) == gold[key].tolist()
        assert detect.nms(d, thr) == gold[key].tolist()
    assert detect.nms(np.zeros((0, 5), np.float32), 0.3) == []
    two = np.array([[0, 0, 9, 9, 0.9], [5, 0, 14, 9, 0.8]], np.float32)
    thr = float(np.float32(50.0) / np.float32(150.0))
    assert detect.cpu_nms(two, thr) == [0] and detect.py_cpu_nms(two, thr) == [0, 1]


@pytest.mark.parametrize('n', [1, 63, 64, 65, 1000, 5000])
def test_nms_random_sizes_vs_oracle(n, dev):
    rng = np.random.default_rng(n)
    c = rng.uniform(0, 600, (n, 2))
    wh = rng.uniform(10, 120, (n, 2))
    # quantised coordinates: many overlaps land exactly on representable ratios, exercising the >= / > conventions
    d = np.hstack([np.round(c - wh / 2), np.round(c + wh / 2), (rng.permutation(n)[:, None] + 1) / (n + 1.0)]).astype(np.float32)
    for mode, ge in ((_lib.NMS_CPU_NMS, True), (_lib.NMS_PY_CPU_NMS, False)):
        order = d[:, 4].argsort()[::-1]
        got = order[_nms_dev(d[order], 0.3, mode, dev)]
        assert got.tolist() == rp.cpu_nms(d, 0.3, ge=ge)
    assert order[_nms_dev(d[order], 0.3, _lib.NMS_PY_CPU_NMS, dev)].tolist() == rp.py_cpu_nms(d, 0.3)


def test_decode_and_detector_chain(gold, dev):
    h, w = gold['fb_image'].shape[:2]
    assert detect.num_priors(h, w) == gold['fb_loc'].shape[0]
    loc = torch.from_numpy(gold['fb_loc']).to(dev)
    for tag in ('net', 'rnd'):
        conf = torch.from_numpy(gold[f'fb_{tag}_conf']).to(dev)
        dets, n = detect.decode_device(loc, conf, h, w)
        n = int(n.item())
        want = gold[f'fb_{tag}_dets_sorted']
        assert n == want.shape[0]
        got = dets[:n].cpu().numpy()
        if n:
            assert np.array_equal(got[:, 4], want[:, 4])                       # scores and their order: exact
            assert np.allclose(got[:, :4], want[:, :4], rtol=2e-6, atol=2e-5)   # exp() is a library call on both sides
            keep, nk = detect.nms_device(dets, 0.3, _lib.NMS_PY_CPU_NMS, n=n)
            assert keep[:int(nk.item())].cpu().numpy().tolist() == rp.py_cpu_nms(got, 0.3)
        final = np.array(detect.detect_postprocess(gold['fb_loc'], gold[f'fb_{tag}_conf'], h, w), np.float32).reshape(-1, 5)
        ref_final = gold[f'fb_{tag}_final']
        assert final.shape == ref_final.shape
        if final.size:
            assert np.array_equal(final[:, 4], ref_final[:, 4]) and np.allclose(final[:, :4], ref_final[:, :4], rtol=2e-6, atol=2e-5)
    # top_k truncation and a rescaled image (FaceBoxes.py:63-79: boxes / scale)
    conf = torch.from_numpy(gold['fb_rnd_conf']).to(dev)
    dets, n = detect.decode_device(loc, conf, h, w, scale=0.5, k=100)
    want = rp.faceboxes_dets(gold['fb_loc'], gold['fb_rnd_conf'], h, w, scale=0.5, top_k=100)
    assert int(n.item()) == 100 and np.array_equal(dets.cpu().numpy()[:, 4], want[:, 4])
    assert np.allclose(dets.cpu().numpy()[:, :4], want[:, :4], rtol=2e-6, atol=2e-5)


def test_prior_boxes_bit_exact_via_zero_offsets(gold, dev):
    """loc = 0 decodes to the priors themselves (exp(0) = 1): corner form of the reference's prior table, exactly."""
    for (h, w) in ((96, 160), (250, 333)):
        pri = gold[f'priors_{h}x{w}']
        p = pri.shape[0]
        conf = torch.zeros((p, 2), device=dev)
        conf[:, 1] = torch.linspace(0.9, 0.1, p, device=dev)                  # descending: rank = prior index
        dets, n = detect.decode_device(torch.zeros((p, 4), device=dev), conf, h, w, k=p)
        assert int(n.item()) == p
        x1y1 = pri[:, :2] - pri[:, 2:] / np.float32(2)
        want = np.hstack([x1y1, pri[:, 2:] + x1y1]) * np.array([w, h, w, h], np.float32)
        assert np.array_equal(dets.cpu().numpy()[:, :4], want.astype(np.float32))
