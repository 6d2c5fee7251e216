"""The frame-axis overlay on the H100: ``Sim3DR.render_batch`` / ``MeshRenderer.render_frames`` and the models'
``overlay_batch`` against the per-frame calls they replace (``Sim3DR.render`` on each frame, after ``get_all_outputs``),
bit for bit for the blended image and the solid overlay.  ``Sim3DR.render`` itself is held to the reference's rasteriser
and cv2 by test_gpu_render.py; the blend's arithmetic is held to cv2 for every byte pair by
test_render_frames_emulation.py."""
import numpy as np
import pytest
import torch

from oracle import synth_model, synth_resnet
from oracle.stage_check import make_model
from synergynet_b200 import Sim3DR, _lib, render, synthetic
from synergynet_b200.inference import RENDER_CFG

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
TRI = synthetic.make_render_topology()
POOL = 20


@pytest.fixture(scope='module')
def pools():
    """Per frame size, POOL full-size meshes (53 215 vertices, 105 408 triangles) scattered over the frame."""
    out = {}
    for h, w in ((720, 1080), (481, 643)):
        out[(h, w)] = synthetic.make_render_meshes(POOL, h, w, seed=h + w, size=min(h, w) / 4.0)
    return out


def _scene(n, h, w, pool, seed):
    """n frames and their mesh lists: 0..16 meshes per frame (frame 1 none), overlapping meshes, in every frame with
    meshes one partly off the canvas and, from 3 meshes on, one wholly off it."""
    rng = np.random.default_rng(seed)
    frames = np.stack([synthetic.make_scene_u8(h, w, seed + 31 * i) for i in range(n)])
    vers = []
    for f in range(n):
        k = 0 if f == 1 else (16 if f == 0 else int(rng.integers(0, 17)))
        lst = []
        for j in range(k):
            v = pool[int(rng.integers(0, POOL))].copy()
            if j == 0:
                v[0] -= 0.45 * w                                           # partly off the left edge
            elif j == 2:
                v[1] += 2.0 * h                                            # wholly below the frame
            elif j % 4 == 3:
                v[:2] = v[:2] * 0.5 + pool[0][:2, :1] * 0.5                # pulled towards the first mesh: overlaps
            lst.append(v)
        vers.append(lst)
    return frames, vers


def _per_frame(frames, vers, alpha, tex):
    out = []
    for f in range(frames.shape[0]):
        if vers[f]:
            out.append(Sim3DR.render(frames[f].copy(), vers[f], TRI, alpha=alpha, tex=tex))
        else:                                                              # the reference's render(img, []): nothing drawn
            out.append((cv2.addWeighted(frames[f], 1 - alpha, frames[f], alpha, 0), frames[f].copy()))
    return out


CASES = [(1, 720, 1080, False, 0.6), (3, 481, 643, True, 0.1), (3, 720, 1080, False, 0.1), (16, 720, 1080, True, 0.6),
         (16, 481, 643, False, 0.1), (64, 720, 1080, False, 0.6), (64, 481, 643, True, 0.1)]


@pytest.mark.parametrize('n,h,w,with_tex,alpha', CASES, ids=[f'{n}x{h}x{w}-{"tex" if t else "light"}-{a}' for n, h, w, t, a in CASES])
def test_render_batch_equals_render_per_frame(pools, n, h, w, with_tex, alpha):
    frames, vers = _scene(n, h, w, pools[(h, w)], seed=n * 7 + h)
    tex = np.random.default_rng(5).uniform(0.2, 1.0, (synthetic.NVER, 3)).astype(np.float32) if with_tex else None
    got = Sim3DR.render_batch(list(frames), vers, TRI, alpha=alpha, tex=tex)
    want = _per_frame(frames, vers, alpha, tex)
    assert len(got) == n
    for f in range(n):
        assert np.array_equal(got[f][1], want[f][1]), f'overlap of frame {f} ({len(vers[f])} meshes)'
        assert np.array_equal(got[f][0], want[f][0]), f'blended frame {f} ({len(vers[f])} meshes)'
    drawn = [f for f in range(n) if vers[f]]
    assert any((got[f][1] != frames[f]).any() for f in drawn) or not drawn
    if n > 1:
        assert np.array_equal(got[1][1], frames[1])                        # the frame without a mesh


def test_render_batch_without_any_mesh_and_file_writes(tmp_path):
    frames = np.stack([synthetic.make_scene_u8(37, 53, s) for s in range(3)])
    got = Sim3DR.render_batch(frames, [[], [], []], TRI, alpha=0.3, wfps=[str(tmp_path / 'a.png'), None, str(tmp_path / 'c.png')])
    for f in range(3):
        assert np.array_equal(got[f][1], frames[f])
        assert np.array_equal(got[f][0], cv2.addWeighted(frames[f], 0.7, frames[f], 0.3, 0))
    assert np.array_equal(cv2.imread(str(tmp_path / 'c.png')), got[2][0])
    assert np.array_equal(cv2.imread(str(tmp_path / 'a_solid.png')), got[0][1])
    assert not (tmp_path / 'b.png').exists() and len(list(tmp_path.iterdir())) == 4


def test_render_module_batch_writes_what_render_writes(tmp_path, pools):
    frames, vers = _scene(3, 481, 643, pools[(481, 643)], seed=2)
    conn = TRI.T
    got = render.render_batch(frames, vers, alpha=0.6, wfps=[str(tmp_path / f'b{i}.png') for i in range(3)], connectivity=conn)
    for f in range(3):
        if vers[f]:
            want = render.render(frames[f].copy(), vers[f], alpha=0.6, wfp=str(tmp_path / f'r{f}.png'), connectivity=conn)
            assert np.array_equal(cv2.imread(str(tmp_path / f'r{f}_solid.png')), cv2.imread(str(tmp_path / f'b{f}_solid.png')))
        else:
            want = cv2.addWeighted(frames[f], 0.4, frames[f], 0.6, 0)
        assert np.array_equal(got[f], want) and np.array_equal(cv2.imread(str(tmp_path / f'b{f}.png')), want)


def _box_of(v, tri, h, w):
    """(x0, y0, x1, y1) union of the clamped triangle boxes of one (3,N) mesh, in numpy."""
    x, y = v[0][tri], v[1][tri]
    x0 = np.maximum(np.floor(x.min(1)).astype(np.int64), 0)
    x1 = np.minimum(np.ceil(x.max(1)).astype(np.int64), w - 1)
    y0 = np.maximum(np.floor(y.min(1)).astype(np.int64), 0)
    y1 = np.minimum(np.ceil(y.max(1)).astype(np.int64), h - 1)
    live = (x1 >= x0) & (y1 >= y0)
    if not live.any():
        return [0, 0, -1, -1]
    return [int(x0[live].min()), int(y0[live].min()), int(x1[live].max()), int(y1[live].max())]


def test_plan_key_total_is_the_clipped_box_area(pools):
    """64 frames x 16 faces at 720 x 1080: the key workspace is the sum of the clipped boxes, a small fraction of the
    B x H x W keys a full canvas per mesh would take."""
    h, w = 720, 1080
    pool = pools[(h, w)]
    rng = np.random.default_rng(11)
    idx = rng.integers(0, POOL, 64 * 16)
    ver = pool[idx].copy()
    ver[::16, 0] -= 0.45 * w                                              # one mesh per frame partly off the canvas
    ver[1::16, 1] += 2.0 * h                                              # and one wholly off it
    r = Sim3DR._renderer_for(TRI, synthetic.NVER)
    v = torch.from_numpy(ver).to(DEV).transpose(1, 2)
    boxes, key_off = r.plan_frames(v, [16] * 64, h, w)
    boxes, key_off = boxes.cpu().numpy(), key_off.cpu().numpy()
    want_boxes = np.array([_box_of(ver[b], TRI, h, w) for b in range(ver.shape[0])])
    assert np.array_equal(boxes, want_boxes)
    areas = np.where(want_boxes[:, 2] >= want_boxes[:, 0], (want_boxes[:, 2] - want_boxes[:, 0] + 1) * (want_boxes[:, 3] - want_boxes[:, 1] + 1), 0)
    assert key_off.tolist() == np.concatenate([[0], np.cumsum(areas)]).tolist()
    assert (areas[1::16] == 0).all()
    full = ver.shape[0] * h * w
    assert key_off[-1] < 0.1 * full, (int(key_off[-1]), full)
    print(f'keys {int(key_off[-1])} of {full} ({key_off[-1] / full:.3%}): {key_off[-1] * 8 / 2**20:.1f} MiB vs {full * 8 / 2**30:.2f} GiB')


def test_bad_inputs_raise_before_any_launch():
    r = Sim3DR._renderer_for(TRI, synthetic.NVER)
    ver = torch.from_numpy(synthetic.make_render_meshes(3, 64, 80, seed=1)).to(DEV).transpose(1, 2)
    frames = torch.zeros((2, 64, 80, 3), dtype=torch.uint8, device=DEV)
    col = torch.zeros((3, synthetic.NVER, 3), dtype=torch.float32, device=DEV)
    out = torch.full_like(frames, 7)
    n0 = r.launches
    with pytest.raises(ValueError, match='counts must give'):
        r.rasterize_frames(frames, ver, col, [1, 1, 1], out=out)
    with pytest.raises(ValueError, match='counts must give'):
        r.rasterize_frames(frames, ver, col, [4, -1], out=out)
    with pytest.raises(_lib.SynergyLibError, match='must run from 0 to 3 meshes'):
        r.rasterize_frames(frames, ver, col, [1, 1], out=out)
    with pytest.raises(ValueError, match='colors must be'):
        r.rasterize_frames(frames, ver, col[:2], [1, 2], out=out)
    with pytest.raises(ValueError, match='frames must be'):
        r.rasterize_frames(frames.float(), ver, col, [1, 2])
    with pytest.raises(ValueError, match='add_weighted takes'):
        Sim3DR.add_weighted(frames, frames[:1], 0.6)
    with pytest.raises(_lib.SynergyLibError, match='not finite'):
        Sim3DR.add_weighted(frames, frames, float('nan'))
    torch.cuda.synchronize()
    assert r.launches == n0 and bool((out == 7).all())


def test_add_weighted_device_equals_cv2_at_unaligned_sizes():
    """The vector path (16-byte multiples) and the scalar path (odd sizes, offset views)."""
    rng = np.random.default_rng(3)
    for shape in ((1, 1, 3), (7, 13, 3), (481, 643, 3), (4, 720, 1080, 3)):
        a = rng.integers(0, 256, shape, dtype=np.uint8)
        b = rng.integers(0, 256, shape, dtype=np.uint8)
        for alpha in (0.1, 0.6, 1.7):
            got = Sim3DR.add_weighted(torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV), alpha).cpu().numpy()
            assert np.array_equal(got, cv2.addWeighted(a, 1 - alpha, b, alpha, 0)), (shape, alpha)
    flat = torch.from_numpy(rng.integers(0, 256, 4099, dtype=np.uint8)).to(DEV)
    got = Sim3DR.add_weighted(flat[1:4097], flat[3:4099], 0.3).cpu().numpy()
    h = flat.cpu().numpy()
    assert np.array_equal(got.reshape(-1, 1), cv2.addWeighted(h[1:4097].reshape(-1, 1), 0.7, h[3:4099].reshape(-1, 1), 0.3, 0))


# ---- overlay_batch -----------------------------------------------------------------------------------------------------------
RECTS = [[[60.3, 80.1, 200.9, 250.4, 0.98], [250.2, -20.0, 372.6, 140.7, 0.91], [300.0, 150.0, 470.0, 350.0, 0.9]],
         [[10.0, 12.0, 130.0, 160.0, 0.7]],
         [],
         [[200.0, 100.0, 330.0, 260.0, 0.8], [-15.5, 200.2, 120.1, 371.0, 0.6]],
         []]


def _loop(model, frames, rects, alpha, tri, tex=None):
    """What a user writes today: get_all_outputs + Sim3DR.render, frame by frame."""
    out = []
    for f in range(frames.shape[0]):
        _, meshes, _ = model.get_all_outputs(frames[f].copy(), rects=rects[f])
        if meshes:
            out.append(Sim3DR.render(frames[f].copy(), meshes, tri, alpha=alpha, tex=tex, cfg=RENDER_CFG))
        else:
            out.append((cv2.addWeighted(frames[f], 1 - alpha, frames[f], alpha, 0), frames[f].copy()))
    return out


def _same(blended, solid, want, where):
    for f, (wb, ws) in enumerate(want):
        assert np.array_equal(solid[f], ws), f'{where}: solid overlay of frame {f}'
        assert np.array_equal(blended[f], wb), f'{where}: blended frame {f}'


@pytest.mark.parametrize('arch', ['mobilenet_v2', 'resnet18'])
def test_overlay_batch_equals_get_all_outputs_and_render_per_frame(synth_pack, arch):
    model = make_model(synth_model.build_state_dict(0)) if arch == 'mobilenet_v2' else \
        make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
    frames = np.stack([synthetic.make_scene_u8(360, 480, 17 + 5 * i) for i in range(5)])
    conn = TRI.T
    blended, solid = model.overlay_batch(list(frames), rects=RECTS, alpha=0.6, connectivity=conn)
    assert blended.shape == solid.shape == frames.shape and blended.dtype == np.uint8
    want = _loop(model, frames, RECTS, 0.6, TRI)
    _same(blended, solid, want, arch)
    assert (solid[0] != frames[0]).any() and np.array_equal(solid[2], frames[2])
    # dense meshes in chunks of two faces: frame 0's three faces are drawn by two calls onto the same canvas
    model.dense_chunk_bytes = 2 * 3 * 4 * synthetic.NVER
    try:
        cb, cs = model.overlay_batch(frames, rects=RECTS, alpha=0.6, connectivity=conn)
        one = model.overlay_batch(frames, rects=RECTS, alpha=0.1, connectivity=conn)
        model.dense_chunk_bytes = 1
        single = model.overlay_batch(frames, rects=RECTS, alpha=0.6, connectivity=conn)
    finally:
        del model.dense_chunk_bytes
    assert np.array_equal(cb, blended) and np.array_equal(cs, solid)
    assert np.array_equal(single[0], blended) and np.array_equal(single[1], solid)
    _same(*one, _loop(model, frames, RECTS, 0.1, TRI), f'{arch} alpha 0.1 chunked')
    # a CUDA stack in, CUDA stacks out
    tb, ts = model.overlay_batch(torch.from_numpy(frames).to(DEV), rects=RECTS, alpha=0.6, connectivity=conn)
    assert tb.is_cuda and ts.is_cuda and np.array_equal(tb.cpu().numpy(), blended) and np.array_equal(ts.cpu().numpy(), solid)
    # no face anywhere
    nb, ns = model.overlay_batch(frames[:2], rects=[[], []], alpha=0.6)
    assert np.array_equal(ns, frames[:2])
    assert all(np.array_equal(nb[f], cv2.addWeighted(frames[f], 0.4, frames[f], 0.6, 0)) for f in range(2))


def test_overlay_batch_default_triangles_and_texture(synth_pack):
    """The model's own triangles (the parameter pack's tri.mat, laid out as render.render lays it out) and a texture."""
    model = make_model(synth_model.build_state_dict(0))
    frames = np.stack([synthetic.make_scene_u8(240, 320, 3 + i) for i in range(2)])
    rects = [[[40.0, 30.0, 120.0, 130.0, 0.9]], [[150.0, 60.0, 230.0, 170.0, 0.8], [10.0, 100.0, 80.0, 190.0, 0.7]]]
    tri = np.ascontiguousarray((np.asarray(synth_pack.tri) - 1).T).astype(np.int32)
    tex = np.random.default_rng(2).uniform(0.3, 1.0, (synthetic.NVER, 3)).astype(np.float32)
    blended, solid = model.overlay_batch(frames, rects=rects, alpha=0.6, tex=tex)
    _same(blended, solid, _loop(model, frames, rects, 0.6, tri, tex), 'default triangles, texture')


def test_overlay_batch_leaves_the_models_outputs_unchanged(synth_pack):
    model = make_model(synth_model.build_state_dict(0))
    frames = np.stack([synthetic.make_scene_u8(360, 480, 40 + i) for i in range(5)])
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(8, seed=9)).to(DEV)
    p0, l0 = model.forward_test(x).clone(), model.forward_landmarks(x).clone()
    g0 = model.get_all_outputs_batch(frames, rects=RECTS)
    model.overlay_batch(frames, rects=RECTS, connectivity=TRI.T)
    assert torch.equal(model.forward_test(x), p0) and torch.equal(model.forward_landmarks(x), l0)
    g1 = model.get_all_outputs_batch(frames, rects=RECTS)
    for (la, ma, pa), (lb, mb, pb) in zip(g0, g1):
        assert all(np.array_equal(a, b) for a, b in zip(la, lb)) and all(np.array_equal(a, b) for a, b in zip(ma, mb))
        assert all(a[0] == b[0] and np.array_equal(a[1], b[1]) for a, b in zip(pa, pb))
    eng = model._engine(DEV)
    assert eng.poll_error() == 0
