"""The image-list overlay on the H100: ``Sim3DR.render_images`` / ``MeshRenderer.render_images`` and the models'
``overlay_images`` against the per-image calls they replace (``Sim3DR.render`` on each image, after ``get_all_outputs``),
bit for bit for the blended image and the solid overlay.  ``Sim3DR.render`` itself is held to the reference's rasteriser
and cv2 by test_gpu_render.py, so this ties the image list to the reference.  Also the plan's key count, in-place drawing
on a slice of a pack, stale and poisoned memory (the protocol of test_gpu_poison.py) and refusals that launch nothing."""
import contextlib

import numpy as np
import pytest
import torch

from oracle import synth_mbv1, synth_model, synth_resnet
from oracle.stage_check import make_model
from synergynet_b200 import Sim3DR, _lib, faceboxes, render, synthetic
from synergynet_b200.inference import RENDER_CFG, ImagePack, pack_images

cv2 = pytest.importorskip('cv2')
pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
TRI = synthetic.make_render_topology()

# (h, w, meshes): 1 x 1, 1 x W, H x 1, odd sizes, a 300 x 400 image with a mesh wholly off it but inside its larger
# neighbours' extent, one image with many meshes, 1080 x 1920, and images without a mesh
SIZES = [(1, 1, 2), (1, 257, 0), (193, 1, 3), (37, 91, 4), (300, 400, 6), (720, 1080, 24), (1080, 1920, 3), (481, 643, 0)]


def _scene(sizes, seed):
    """Images and their mesh lists.  From 4 meshes on, the first four cross the left, right, top and bottom edge of their
    own image; the 300 x 400 image's sixth mesh lies wholly right of and below it, inside the 720 x 1080 extent."""
    images, vers = [], []
    for i, (h, w, k) in enumerate(sizes):
        images.append(synthetic.make_scene_u8(h, w, seed + 13 * i))
        v = synthetic.make_render_meshes(max(k, 1), h, w, seed=seed + i, size=max(4.0, min(h, w) / 4.0))[:k].copy()
        if k >= 4:
            v[0, 0] -= 0.45 * w
            v[1, 0] += 0.45 * w
            v[2, 1] -= 0.45 * h
            v[3, 1] += 0.45 * h
        if (h, w) == (300, 400):
            v[5, 0] += w + 40.0
            v[5, 1] += h + 40.0
        vers.append(list(v))
    return images, vers


def _per_image(images, vers, alpha, tex):
    out = []
    for im, vl in zip(images, vers):
        if vl:
            out.append(Sim3DR.render(im.copy(), vl, TRI, alpha=alpha, tex=tex))
        else:                                                              # the reference's render(img, []): nothing drawn
            out.append((cv2.addWeighted(im, 1 - alpha, im, alpha, 0), im.copy()))
    return out


CASES = [(False, 0.6), (True, 0.3), (False, 0.3), (True, 0.6)]


@pytest.mark.parametrize('with_tex,alpha', CASES, ids=[f'{"tex" if t else "light"}-{a}' for t, a in CASES])
def test_render_images_equals_render_per_image(with_tex, alpha):
    images, vers = _scene(SIZES, seed=3)
    tex = np.random.default_rng(5).uniform(0.2, 1.0, (synthetic.NVER, 3)).astype(np.float32) if with_tex else None
    got = Sim3DR.render_images(images, vers, TRI, alpha=alpha, tex=tex)
    want = _per_image(images, vers, alpha, tex)
    assert len(got) == len(images)
    for i, ((gb, gs), (wb, ws)) in enumerate(zip(got, want)):
        assert gs.shape == images[i].shape and gb.dtype == np.uint8
        assert np.array_equal(gs, ws), f'overlap of image {i} {images[i].shape} ({len(vers[i])} meshes)'
        assert np.array_equal(gb, wb), f'blended image {i} {images[i].shape} ({len(vers[i])} meshes)'
    for i, (h, w, k) in enumerate(SIZES):
        if k == 0:
            assert np.array_equal(got[i][1], images[i])
        elif h > 1 and w > 1:
            assert (got[i][1] != images[i]).any(), i
    # the mesh wholly off the 300 x 400 image draws nothing there: without it, the same bytes
    j = [s[:2] for s in SIZES].index((300, 400))
    alone = Sim3DR.render(images[j].copy(), vers[j][:5], TRI, alpha=alpha, tex=tex)
    assert np.array_equal(got[j][1], alone[1]) and np.array_equal(got[j][0], alone[0])


def test_render_images_module_twin_and_file_writes(tmp_path):
    images, vers = _scene(SIZES[:5], seed=8)
    wfps = [str(tmp_path / f'i{i}.png') if i % 2 == 0 else None for i in range(5)]
    got = render.render_images(images, vers, alpha=0.6, wfps=wfps, connectivity=TRI.T)
    for i in range(5):
        want = render.render(images[i].copy(), vers[i], alpha=0.6, connectivity=TRI.T) if vers[i] else \
            cv2.addWeighted(images[i], 0.4, images[i], 0.6, 0)
        assert np.array_equal(got[i], want), i
        if wfps[i]:
            assert np.array_equal(cv2.imread(wfps[i]), want)
    assert len(list(tmp_path.iterdir())) == 6


def test_equal_sizes_equal_render_batch():
    images, vers = _scene([(481, 643, k) for k in (5, 0, 2, 7)], seed=21)
    got = Sim3DR.render_images(images, vers, TRI, alpha=0.6)
    batch = Sim3DR.render_batch(np.stack(images), vers, TRI, alpha=0.6)
    for i in range(4):
        assert np.array_equal(got[i][0], batch[i][0]) and np.array_equal(got[i][1], batch[i][1]), i
    none = Sim3DR.render_images(images[:2], [[], []], TRI, alpha=0.3)
    assert all(np.array_equal(none[i][1], images[i]) for i in range(2))


def _box_of(v, h, w):
    """(x0, y0, x1, y1) union of the clamped triangle boxes of one (3,N) mesh on an h x w image, in numpy."""
    x, y = v[0][TRI], v[1][TRI]
    x0 = np.maximum(np.floor(x.min(1)).astype(np.int64), 0)
    x1 = np.minimum(np.ceil(x.max(1)).astype(np.int64), w - 1)
    y0 = np.maximum(np.floor(y.min(1)).astype(np.int64), 0)
    y1 = np.minimum(np.ceil(y.max(1)).astype(np.int64), h - 1)
    live = (x1 >= x0) & (y1 >= y0)
    if not live.any():
        return [0, 0, -1, -1]
    return [int(x0[live].min()), int(y0[live].min()), int(x1[live].max()), int(y1[live].max())]


def _device_scene(sizes, seed):
    images, vers = _scene(sizes, seed)
    counts = [len(v) for v in vers]
    ver = np.stack([m for vl in vers for m in vl])
    return images, vers, counts, ver, torch.from_numpy(ver).to(DEV).transpose(1, 2)


def test_plan_key_total_is_each_box_clamped_to_its_own_image():
    images, vers, counts, ver, v = _device_scene(SIZES, seed=4)
    r = Sim3DR._renderer_for(TRI, synthetic.NVER)
    boxes, key_off = r.plan_images(pack_images(images, DEV), v, counts)
    boxes, key_off = boxes.cpu().numpy(), key_off.cpu().numpy()
    own = [(h, w) for h, w, k in SIZES for _ in range(k)]
    want = np.array([_box_of(ver[b], *own[b]) for b in range(ver.shape[0])])
    assert np.array_equal(boxes, want)
    areas = np.where(want[:, 2] >= want[:, 0], (want[:, 2] - want[:, 0] + 1) * (want[:, 3] - want[:, 1] + 1), 0)
    assert key_off.tolist() == np.concatenate([[0], np.cumsum(areas)]).tolist()
    off_own = sum(k for h, w, k in SIZES[:4]) + 5                      # the 300 x 400 image's mesh off it
    assert areas[off_own] == 0 and _box_of(ver[off_own], 720, 1080)[2] >= 0
    padded = ver.shape[0] * max(h for h, w, k in SIZES) * max(w for h, w, k in SIZES)
    print(f'keys {int(key_off[-1])} ({key_off[-1] * 8 / 2**20:.1f} MiB) vs {padded * 8 / 2**30:.2f} GiB padded to the largest image')


def test_in_place_on_a_slice_writes_nothing_outside_it():
    sizes = [(37, 91, 2), (1, 1, 2), (300, 400, 6), (193, 1, 3), (1, 257, 2)]
    images, vers = _scene(sizes, seed=9)
    # the slice's meshes include, for the 1 x 1 and 193 x 1 images, meshes larger than both neighbours' extents
    pack = pack_images(images, DEV)
    before = pack.data.clone()
    r = Sim3DR._renderer_for(TRI, synthetic.NVER)
    part = pack.slice(1, 4)
    sub = [m for vl in vers[1:4] for m in vl]
    v = torch.from_numpy(np.stack(sub)).to(DEV).transpose(1, 2)
    col = r.colors(v, r.normals(v), Sim3DR._light_cfg(**RENDER_CFG))
    assert r.rasterize_images(part, v, col, [len(x) for x in vers[1:4]], out=part) is part
    a, b = pack.offsets[1], pack.offsets[4]
    after = pack.data
    assert torch.equal(after[:a], before[:a]) and torch.equal(after[b:], before[b:])
    want = _per_image(images[1:4], vers[1:4], 0.6, None)
    for i in range(3):
        assert np.array_equal(pack.image(1 + i).cpu().numpy(), want[i][1]), i


# ---- overlay_images --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def fb():
    return faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0), device='cuda:0')


def _checkpoint(arch):
    if arch == 'mobilenet_v2':
        return make_model(synth_model.build_state_dict(0))
    if arch.startswith('resnet'):
        return make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
    return make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)


IMAGE_SIZES = [(360, 480), (250, 333), (1, 1), (720, 1080), (97, 61)]
IMAGE_RECTS = [[[60.3, 80.1, 200.9, 250.4, 0.98], [250.2, -20.0, 372.6, 140.7, 0.91], [300.0, 150.0, 470.0, 350.0, 0.9]],
               [[-15.5, 100.2, 120.1, 271.0, 0.6]],
               [],
               [[500.0, 300.0, 800.0, 620.0, 0.9], [950.0, 600.0, 1150.0, 790.0, 0.8]],
               [[10.0, 12.0, 70.0, 90.0, 0.7]]]


def _loop(model, images, rects, alpha, tri, tex=None):
    """What a user writes today: get_all_outputs + Sim3DR.render, image by image."""
    out = []
    for im, rc in zip(images, rects):
        _, meshes, _ = model.get_all_outputs(im.copy(), rects=rc)
        if meshes:
            out.append(Sim3DR.render(im.copy(), meshes, tri, alpha=alpha, tex=tex, cfg=RENDER_CFG))
        else:
            out.append((cv2.addWeighted(im, 1 - alpha, im, alpha, 0), im.copy()))
    return out


def _same(got, want, where):
    blended, solid = got
    assert len(blended) == len(solid) == len(want), where
    for i, (wb, ws) in enumerate(want):
        gs = solid[i].cpu().numpy() if isinstance(solid[i], torch.Tensor) else solid[i]
        gb = blended[i].cpu().numpy() if isinstance(blended[i], torch.Tensor) else blended[i]
        assert np.array_equal(gs, ws), f'{where}: solid overlay of image {i}'
        assert np.array_equal(gb, wb), f'{where}: blended image {i}'


@pytest.mark.parametrize('arch', ['mobilenet_v2', 'resnet18', 'mobilenet_05'])
def test_overlay_images_equals_get_all_outputs_and_render_per_image(synth_pack, fb, arch):
    model = _checkpoint(arch)
    images = [synthetic.make_scene_u8(h, w, 17 + 5 * i) for i, (h, w) in enumerate(IMAGE_SIZES)]
    conn = TRI.T
    got = model.overlay_images(images, rects=IMAGE_RECTS, alpha=0.6, connectivity=conn)
    assert all(isinstance(x, np.ndarray) and x.shape == im.shape for x, im in zip(got[0] + got[1], images + images))
    want = _loop(model, images, IMAGE_RECTS, 0.6, TRI)
    _same(got, want, arch)
    assert (got[1][0] != images[0]).any() and np.array_equal(got[1][2], images[2])
    for i in range(len(images)):                                    # and overlay_batch on the one-image stack
        ob, os_ = model.overlay_batch(images[i][None], rects=[IMAGE_RECTS[i]], alpha=0.6, connectivity=conn)
        assert np.array_equal(ob[0], got[0][i]) and np.array_equal(os_[0], got[1][i]), f'{arch} overlay_batch of image {i}'
    # dense meshes in chunks of two faces (a chunk ends inside image 0 and another spans images 0 and 1), then of one
    model.dense_chunk_bytes = 2 * 3 * 4 * synthetic.NVER
    try:
        two = model.overlay_images(images, rects=IMAGE_RECTS, alpha=0.6, connectivity=conn)
        low = model.overlay_images(images, rects=IMAGE_RECTS, alpha=0.3, connectivity=conn)
        model.dense_chunk_bytes = 1
        one = model.overlay_images(images, rects=IMAGE_RECTS, alpha=0.6, connectivity=conn)
    finally:
        del model.dense_chunk_bytes
    _same(two, want, f'{arch} chunks of two')
    _same(one, want, f'{arch} chunks of one')
    _same(low, _loop(model, images, IMAGE_RECTS, 0.3, TRI), f'{arch} alpha 0.3 chunked')
    # CUDA tensors in, CUDA views out
    dev = model.overlay_images([torch.from_numpy(im).to(DEV) for im in images], rects=IMAGE_RECTS, alpha=0.6, connectivity=conn)
    assert all(isinstance(t, torch.Tensor) and t.is_cuda for t in dev[0] + dev[1])
    _same(dev, want, f'{arch} CUDA inputs')
    # no face anywhere
    nb, ns = model.overlay_images(images[:3], rects=[[], [], []], alpha=0.6)
    assert all(np.array_equal(ns[i], images[i]) for i in range(3))
    assert all(np.array_equal(nb[i], cv2.addWeighted(images[i], 0.4, images[i], 0.6, 0)) for i in range(3))
    # rects=None: the detector's detect_images takes the upload
    model.face_detector = fb
    try:
        small = [synthetic.make_scene_u8(h, w, 3 + h) for h, w in ((240, 320), (300, 200), (1, 1))]
        auto = model.overlay_images(small, alpha=0.6, connectivity=conn)
        rects = fb.detect_images(small)
        _same(auto, _loop(model, small, rects, 0.6, TRI), f'{arch} detected')
    finally:
        model.face_detector = None


def test_overlay_images_default_triangles_and_texture(synth_pack):
    model = _checkpoint('mobilenet_v2')
    images = [synthetic.make_scene_u8(240, 320, 3), synthetic.make_scene_u8(131, 203, 4)]
    rects = [[[40.0, 30.0, 120.0, 130.0, 0.9]], [[150.0, 60.0, 230.0, 170.0, 0.8], [10.0, 40.0, 80.0, 130.0, 0.7]]]
    tri = np.ascontiguousarray((np.asarray(synth_pack.tri) - 1).T).astype(np.int32)
    tex = np.random.default_rng(2).uniform(0.3, 1.0, (synthetic.NVER, 3)).astype(np.float32)
    _same(model.overlay_images(images, rects=rects, alpha=0.6, tex=tex), _loop(model, images, rects, 0.6, tri, tex), 'texture')


def test_overlay_images_leaves_the_models_outputs_unchanged(synth_pack):
    model = _checkpoint('mobilenet_v2')
    images = [synthetic.make_scene_u8(h, w, 40 + i) for i, (h, w) in enumerate(IMAGE_SIZES)]
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(8, seed=9)).to(DEV)
    p0, l0 = model.forward_test(x).clone(), model.forward_landmarks(x).clone()
    g0 = model.get_all_outputs_images(images, rects=IMAGE_RECTS)
    model.overlay_images(images, rects=IMAGE_RECTS, connectivity=TRI.T)
    assert torch.equal(model.forward_test(x), p0) and torch.equal(model.forward_landmarks(x), l0)
    g1 = model.get_all_outputs_images(images, rects=IMAGE_RECTS)
    for (la, ma, pa), (lb, mb, pb) in zip(g0, g1):
        assert all(np.array_equal(a, b) for a, b in zip(la, lb)) and all(np.array_equal(a, b) for a, b in zip(ma, mb))
        assert all(a[0] == b[0] and np.array_equal(a[1], b[1]) for a, b in zip(pa, pb))
    assert model._engine(DEV).poll_error() == 0


# ---- stale and poisoned memory (the protocol of test_gpu_poison.py) -----------------------------------------------------------
FILLS = (0xFF, 0x7F)


@contextlib.contextmanager
def poisoned_empty(byte: int, int_byte: int):
    """Every tensor ``torch.empty`` / ``empty_like`` / ``empty_strided`` returns is filled with ``byte`` (floating-point,
    uint8) or ``int_byte`` (integer dtypes)."""
    orig = {n: getattr(torch, n) for n in ('empty', 'empty_like', 'empty_strided')}

    def wrap(fn):
        def poisoned(*args, **kwargs):
            t = fn(*args, **kwargs)
            if t.numel():
                t.untyped_storage().fill_(byte if t.dtype.is_floating_point or t.dtype == torch.uint8 else int_byte)
            return t
        return poisoned

    with pytest.MonkeyPatch.context() as mp:
        for name, fn in orig.items():
            mp.setattr(torch, name, wrap(fn))
        yield


def _bits(out):
    """The bytes of every tensor of a (nested) result, on the host."""
    if isinstance(out, ImagePack):
        return [out.data.cpu().numpy().copy()]
    if isinstance(out, torch.Tensor):
        return [out.contiguous().view(torch.uint8).cpu().numpy().copy()]
    if isinstance(out, np.ndarray):
        return [out.copy()]
    return [b for o in out for b in _bits(o)]


def _check(cases, r0, int_byte, fill=(), engines=()):
    """Stale, then poisoned under each fill: every case must return the clean bits."""
    def expect(tag, got, want):
        torch.cuda.synchronize()
        assert len(got) == len(want) and all(np.array_equal(g, w) for g, w in zip(got, want)), tag
        for e in engines:
            assert e.poll_error() == 0, f'{tag}: error flag raised'

    for name, fn in cases.items():
        expect(f'{name} stale', _bits(fn()), r0[name])
    for name, fn in cases.items():
        for byte in FILLS:
            for h in fill:
                h.debug_fill_workspaces(byte)
            with poisoned_empty(byte, byte if int_byte is None else int_byte):
                got = _bits(fn())
            expect(f'{name} fill 0x{byte:02X}', got, r0[name])


def test_stale_and_poisoned_memory(synth_pack):
    """The key workspace is cleared before the depth pass, the boxes before the box pass, and the scan writes every key
    offset, so the render cases take the fill in their integer buffers too (keys, boxes, key offsets)."""
    r = Sim3DR._renderer_for(TRI, synthetic.NVER)
    sizes = [(1, 1, 1), (37, 91, 4), (1, 257, 0), (120, 160, 5), (193, 1, 2)]
    images, vers, counts, ver, v = _device_scene(sizes, seed=31)
    pack = pack_images(images, DEV)
    col = r.colors(v, r.normals(v), Sim3DR._light_cfg(**RENDER_CFG))
    cases = {
        'plan_images': lambda: r.plan_images(pack, v, counts),
        'rasterize_images': lambda: r.rasterize_images(pack, v, col, counts),
        'render_images': lambda: r.render_images(pack, v, counts, Sim3DR._light_cfg(**RENDER_CFG), None, 0.6),
    }
    model = _checkpoint('mobilenet_v2')
    eng = model._engine(DEV)
    oimages = [synthetic.make_scene_u8(h, w, 50 + i) for i, (h, w) in enumerate(IMAGE_SIZES)]
    model.dense_chunk_bytes = 2 * 3 * 4 * synthetic.NVER
    try:
        ocases = {'overlay_images': lambda: model.overlay_images(oimages, rects=IMAGE_RECTS, alpha=0.6, connectivity=TRI.T)}
        r0 = {n: _bits(fn()) for n, fn in {**cases, **ocases}.items()}
        # the larger calls: more and larger images, more meshes, more faces
        big_images, _, big_counts, _, big_v = _device_scene([(300, 400, 6), (720, 1080, 12), (37, 91, 4)], seed=32)
        big_pack = pack_images(big_images, DEV)
        r.render_images(big_pack, big_v, big_counts)
        model.overlay_images([synthetic.make_scene_u8(720, 1080, 60 + i) for i in range(3)],
                             rects=[IMAGE_RECTS[0] + IMAGE_RECTS[3]] * 3, connectivity=TRI.T)
        _check(cases, r0, int_byte=None)
        _check(ocases, r0, int_byte=0, fill=(eng,), engines=(eng,))
    finally:
        del model.dense_chunk_bytes


# ---- refusals ----------------------------------------------------------------------------------------------------------------
def test_bad_inputs_raise_before_any_launch(synth_pack):
    r = Sim3DR._renderer_for(TRI, synthetic.NVER)
    images, vers, counts, ver, v = _device_scene([(64, 80, 2), (30, 50, 1)], seed=1)
    pack = pack_images(images, DEV)
    col = torch.zeros((3, synthetic.NVER, 3), dtype=torch.float32, device=DEV)
    out = ImagePack(torch.full_like(pack.data, 7), pack.sizes)
    torch.cuda.synchronize()
    n0 = r.launches
    with pytest.raises(ValueError, match='counts must give'):
        r.rasterize_images(pack, v, col, [1, 1, 1], out=out)
    with pytest.raises(ValueError, match='counts must give'):
        r.rasterize_images(pack, v, col, [4, -1], out=out)
    with pytest.raises(_lib.SynergyLibError, match='must run from 0 to 3 meshes'):
        r.rasterize_images(pack, v, col, [1, 1], out=out)
    with pytest.raises(ValueError, match='colors must be'):
        r.rasterize_images(pack, v, col[:2], [1, 2], out=out)
    with pytest.raises(ValueError, match='out must be an ImagePack'):
        r.rasterize_images(pack, v, col, [2, 1], out=ImagePack(out.data[:-90], [(64, 80), (30, 49)]))
    with pytest.raises(ValueError, match='images must be an ImagePack'):
        r.rasterize_images(pack.data, v, col, [2, 1])
    with pytest.raises(ValueError, match='counts must give'):
        r.plan_images(pack, v, [3])
    torch.cuda.synchronize()
    assert r.launches == n0 and bool((out.data == 7).all())
    model = _checkpoint('mobilenet_v2')
    eng = model._engine(DEV)
    l0 = eng.launch_count
    with pytest.raises(ValueError, match='1 rect lists for 2 frames'):
        model.overlay_images(images, rects=[[]])
    with pytest.raises(ValueError, match='every image must be'):
        model.overlay_images([images[0], np.zeros((5, 5, 4), np.uint8)], rects=[[], []])
    with pytest.raises(ValueError, match='mesh lists'):
        Sim3DR.render_images(images, vers[:1], TRI)
    torch.cuda.synchronize()
    assert eng.launch_count == l0 and r.launches == n0
