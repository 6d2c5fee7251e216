"""CPU checks of the UV texture path (``UVLayout``, ``syn_uv_sample``, ``syn_mesh_lighting_textures`` and the ``uv_*``
model methods) without a GPU: the texel coordinates and their resolution equal numpy's expressions, a host restatement
of the sampler gives the scripts' colour tables bit for bit, and every refusal comes before any CUDA work."""
import ctypes as C
import types

import numpy as np
import pytest

from synergynet_b200 import _lib, synthetic
from synergynet_b200.inference import UVLayout, uv_maps_host


def _fails(code, want, text):
    assert code == want, (code, _lib.load().syn_last_error())
    assert text in _lib.load().syn_last_error(), _lib.load().syn_last_error()


def sample_host(layout, maps, face_map):
    """The kernel's gather restated: face f reads map face_map[f] at the resolved (row, column) of each kept vertex."""
    tex, col = [], []
    for f in face_map:
        m = maps[f]
        t = layout.texels(m.shape[0], m.shape[1])
        px = m[t[:, 0], t[:, 1], :3]
        tex.append(px.astype(np.float32) / np.float32(255.0))
        col.append(px.astype(np.int64))
    return np.stack(tex), np.stack(col)


def reference_tables(uv, keep, m):
    """artistic.py:49-53,126-131: coord_u / coord_v, then np.flip(map, 0)[coord_u, coord_v][keep]."""
    coord_u = (uv[:, 1] * 255.0).astype(np.int32)
    coord_v = (uv[:, 0] * 255.0).astype(np.int32)
    colors_uv = np.flip(m, axis=0)[coord_u, coord_v, :]
    return colors_uv[keep, :].astype(np.float32) / 255.0, colors_uv[keep, :].astype(np.float32)


def _layout_for(rows, cols, keep=None, tri=None):
    """A layout whose coordinates are the given integers (negative ones included): uv = (c +- 0.5) / 255, truncated back."""
    to_uv = lambda c: (np.asarray(c, np.float64) + np.where(np.asarray(c) < 0, -0.5, 0.5)) / 255.0
    uv = np.stack([to_uv(cols), to_uv(rows)], 1)
    n = len(rows)
    keep = np.arange(n) if keep is None else keep
    tri = np.array([[1], [1], [1]]) if tri is None else tri
    layout = UVLayout(uv, keep, tri)
    assert np.array_equal(layout.coord_u, rows) and np.array_equal(layout.coord_v, cols)
    return uv, layout


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_coordinates_are_numpys(dtype):
    uv, keep, tri = synthetic.make_uv_layout(0, nver=5000, dtype=dtype)
    assert uv.dtype == dtype
    layout = UVLayout(uv, keep, tri)
    assert np.array_equal(layout.coord_u, (uv[:, 1] * 255.0).astype(np.int32))
    assert np.array_equal(layout.coord_v, (uv[:, 0] * 255.0).astype(np.int32))
    assert layout.coord_u.max() == 255 and layout.coord_u.min() == 0
    # the neighbours of k/255 land on both sides of k: the float32 and float64 layouts truncate differently there
    assert np.array_equal(layout.render_tri, (tri - 1).T)
    m = synthetic.make_uv_map(256, 256, seed=1)
    tex, col = reference_tables(uv, keep, m)
    t, c = sample_host(layout, [m], [0])
    assert t.tobytes() == tex.tobytes() and np.array_equal(c[0], col)


@pytest.mark.parametrize('h,w', [(1, 1), (1, 7), (5, 1), (3, 4), (256, 256), (255, 257), (512, 300), (300, 512)])
def test_resolution_equals_flipped_indexing(h, w):
    rng = np.random.default_rng(h * 1000 + w)
    n = 400
    rows = rng.integers(-h, h, n)
    cols = rng.integers(-w, w, n)
    rows[:4] = (-h, h - 1, 0, -1)
    cols[:4] = (w - 1, -w, -1, 0)
    keep = np.sort(rng.choice(n, 300, replace=False))
    uv, layout = _layout_for(rows, cols, keep)
    m = synthetic.make_uv_map(h, w, seed=h + w)
    want = np.flip(m, axis=0)[layout.coord_u, layout.coord_v][keep]
    t = layout.texels(h, w)
    assert t.dtype == np.int32 and t.shape == (300, 2)
    assert (t[:, 0] >= 0).all() and (t[:, 0] < h).all() and (t[:, 1] >= 0).all() and (t[:, 1] < w).all()
    assert np.array_equal(m[t[:, 0], t[:, 1]], want)
    tex, col = reference_tables(uv, keep, m)
    et, ec = sample_host(layout, [m], [0])
    assert et[0].tobytes() == tex.tobytes() and np.array_equal(ec[0].astype(np.float32), col)


def test_out_of_range_coordinate_raises_for_unkept_vertex():
    rows, cols = np.array([0, 1, 2, 9]), np.array([0, 1, 2, 3])
    uv, layout = _layout_for(rows, cols, keep=np.array([0, 1, 2]))
    layout.texels(10, 10)
    with pytest.raises(IndexError, match='vertex 3: index 9 is out of bounds for axis 0 with size 4 of map X'):
        layout.texels(4, 4, 'map X')
    with pytest.raises(IndexError):
        np.flip(np.zeros((4, 4, 3)), 0)[layout.coord_u, layout.coord_v]               # what the reference raises
    _, layout = _layout_for(np.array([0, 0]), np.array([0, -3]))
    with pytest.raises(IndexError, match='vertex 1: index -3 is out of bounds for axis 1 with size 2'):
        layout.texels(2, 2)
    assert np.array_equal(layout.texels(2, 3), [[1, 0], [1, 0]])


def test_layout_refusals():
    uv = np.zeros((10, 2), np.float32)
    tri = np.array([[1], [2], [3]])
    with pytest.raises(ValueError, match='BFM_UV'):
        UVLayout(np.zeros((10, 2), np.int32), np.arange(5), tri)
    with pytest.raises(ValueError, match='BFM_UV'):
        UVLayout(np.zeros(10, np.float32), np.arange(5), tri)
    with pytest.raises(ValueError, match=r'keptInd\[2\] = 10 lies outside \[0, 10\)'):
        UVLayout(uv, np.array([0, 1, 10]), tri)
    with pytest.raises(ValueError, match=r'keptInd\[0\] = -1'):
        UVLayout(uv, np.array([-1, 1]), tri)
    with pytest.raises(ValueError, match='keptInd'):
        UVLayout(uv, np.array([0.0, 1.0]), tri)
    with pytest.raises(ValueError, match='deletedTri must be a'):
        UVLayout(uv, np.arange(5), tri.T)
    with pytest.raises(ValueError, match='deletedTri must be a'):
        UVLayout(uv, np.arange(5), tri.astype(np.float64))
    with pytest.raises(ValueError, match=r'deletedTri\[1, 0\] - 1 = 5 lies outside \[0, 5\)'):
        UVLayout(uv, np.arange(5), np.array([[1], [6], [2]]))
    with pytest.raises(ValueError, match=r'deletedTri\[0, 0\] - 1 = -1'):
        UVLayout(uv, np.arange(5), np.array([[0], [1], [2]]))


def test_map_refusals_and_channels():
    m3 = synthetic.make_uv_map(6, 5, seed=0)
    m4 = synthetic.make_uv_map(6, 5, seed=0, channels=4)
    with pytest.raises(ValueError, match='uint8'):
        uv_maps_host(m3.astype(np.uint16), 1, False)
    with pytest.raises(ValueError, match=r'\(h, w, 3\) or \(h, w, 4\)'):
        uv_maps_host(m3[:, :, 0], 1, False)                                           # grayscale
    with pytest.raises(ValueError, match=r'\(h, w, 3\) or \(h, w, 4\)'):
        uv_maps_host([m3[:, :, :1]], 1, False)
    with pytest.raises(ValueError, match='4-channel UV map cannot texture the overlay'):
        uv_maps_host(m4, 1, True)
    with pytest.raises(ValueError, match='2 UV maps for 3 images'):
        uv_maps_host([m3, m3], 3, False)
    (got,) = uv_maps_host(m4, 1, False)
    assert got.shape == (6, 5, 3) and np.array_equal(got, m4[:, :, :3]) and got.flags.c_contiguous
    assert len(uv_maps_host(m3, 4, True)) == 1 and len(uv_maps_host(np.stack([m3, m3]), 2, True)) == 2
    # channels 2, 1, 0 of a 4-channel map are what write_obj_with_colors prints: dropping channel 3 keeps them
    uv, keep, _ = synthetic.make_uv_layout(1, nver=300)
    _, c4 = reference_tables(uv, keep, synthetic.make_uv_map(256, 256, seed=2, channels=4))
    _, c3 = reference_tables(uv, keep, synthetic.make_uv_map(256, 256, seed=2, channels=4)[:, :, :3])
    assert np.array_equal(c4[:, :3], c3)


def test_sampler_emulation_on_ragged_maps():
    uv, keep, tri = synthetic.make_uv_layout(2, nver=3000)
    layout = UVLayout(uv, keep, tri)
    maps = [synthetic.make_uv_map(h, w, seed=i) for i, (h, w) in enumerate([(256, 256), (300, 512), (512, 300), (257, 256)])]
    face_map = [0, 0, 3, 1, 2, 2, 1]
    tex, col = sample_host(layout, maps, face_map)
    for f, m in enumerate(face_map):
        t, c = reference_tables(uv, keep, maps[m])
        assert tex[f].tobytes() == t.tobytes() and np.array_equal(col[f].astype(np.float32), c)


def test_uv_sample_rejects_bad_arguments():
    lib = _lib.load()
    p = C.c_void_p(8)                                      # never dereferenced: every call below fails validation first
    table = np.ascontiguousarray(np.array([[0, 2, 3], [18, 1, 1]], np.int64))
    texels = np.zeros((2, 4, 2), np.int32)
    fmap = np.array([0, 1, 1], np.int32)

    def call(maps=p, nbytes=21, tb=table, tbd=p, n=2, tx=texels, txd=p, k=4, fm=fmap, fmd=p, f=3, tex=p, col=p):
        return lib.syn_uv_sample(maps, nbytes, None if tb is None else tb.ctypes.data, tbd, n, None if tx is None else tx.ctypes.data,
                                 txd, k, None if fm is None else fm.ctypes.data, fmd, f, tex, col, None)

    for kw in ({'maps': None}, {'tb': None}, {'tbd': None}, {'tx': None}, {'txd': None}, {'fm': None}, {'fmd': None},
               {'tex': None, 'col': None}):
        _fails(call(**kw), 1, b'syn_uv_sample: null pointer')
    _fails(call(txd=C.c_void_p(12)), 1, b'not 8-byte aligned')
    _fails(call(n=0), 1, b'0 maps')
    _fails(call(k=0), 1, b'0 kept vertices')
    _fails(call(f=0), 1, b'0 faces')
    _fails(call(f=65536), 1, b'65536 faces')
    _fails(call(nbytes=-1), 1, b'-1 map bytes')
    _fails(call(nbytes=20), 4, b'map 1 (1x1 at byte 18) does not fit the 20 map bytes')
    _fails(call(tb=np.ascontiguousarray(np.array([[0, 2, 3], [15, 1, 1]], np.int64))), 4, b'does not fit')      # overlap
    _fails(call(tb=np.ascontiguousarray(np.array([[0, 0, 3], [18, 1, 1]], np.int64))), 4, b'map 0 is 0x3')
    bad = texels.copy()
    bad[1, 2] = (1, 0)
    _fails(call(tx=bad), 4, b'texel 2 of map 1 is (1, 0), outside its 1x1')
    bad = texels.copy()
    bad[0, 3] = (0, -1)
    _fails(call(tx=bad), 4, b'texel 3 of map 0 is (0, -1)')
    _fails(call(fm=np.array([0, 2, 1], np.int32)), 4, b'face 1 names map 2 of 2')


def test_lighting_textures_rejects_bad_arguments():
    lib = _lib.load()
    p = C.c_void_p(8)
    cfg = _lib.LightCfg()

    def call(tex=p, ts=30, v=p, nver=10):
        return lib.syn_mesh_lighting_textures(v, 30, 3, 1, 2, nver, p, C.byref(cfg), tex, ts, p, p, None)

    _fails(call(tex=None), 1, b'syn_mesh_lighting_textures: null texture')
    _fails(call(ts=-1), 1, b'texture mesh stride -1')
    _fails(call(ts=29), 1, b'texture mesh stride 29')
    _fails(call(v=None), 1, b'mesh view')


@pytest.fixture()
def cpu_model(synth_pack):
    from synergynet_b200 import model_building
    model = model_building.SynergyNet(types.SimpleNamespace(arch='mobilenet_v2', img_size=120), _device=None)
    model.eval()
    return model


def test_model_refuses_before_cuda(cpu_model, monkeypatch):
    """Every refusal of the uv_* methods comes before the model touches CUDA: launches and device lookups raise here."""
    import torch
    from synergynet_b200 import model_building

    def no_cuda(*a, **k):
        raise AssertionError('CUDA reached before the refusal')

    monkeypatch.setattr(_lib, 'launch', no_cuda)
    monkeypatch.setattr(model_building._SynergyBase, '_frames_front', no_cuda)
    monkeypatch.setattr(torch.Tensor, 'cuda', no_cuda)
    n = cpu_model.u.shape[0] // 3
    layout = UVLayout(*synthetic.make_uv_layout(3, nver=n))
    images = [np.zeros((40, 50, 3), np.uint8), np.zeros((30, 20, 3), np.uint8)]
    m = synthetic.make_uv_map(256, 256)
    roi = [[[0, 0, 20, 20, 1.0]], []]
    for name in ('uv_obj_images', 'uv_overlay_images', 'uv_obj_batch', 'uv_overlay_batch'):
        imgs = images if name.endswith('images') else [images[0], images[0]]
        fn = getattr(cpu_model, name)
        with pytest.raises(ValueError, match='not both'):
            fn(imgs, m, layout, rects=roi, rois=roi)
        with pytest.raises(ValueError, match='give rects or rois'):
            fn(imgs, m, layout)
        with pytest.raises(ValueError, match='uint8'):
            fn(imgs, m.astype(np.uint16), layout, rois=roi)
        with pytest.raises(ValueError, match=r'\(h, w, 3\) or \(h, w, 4\)'):
            fn(imgs, m[:, :, 0], layout, rois=roi)
        with pytest.raises(ValueError, match='3 UV maps for 2 images'):
            fn(imgs, [m, m, m], layout, rois=roi)
        with pytest.raises(ValueError, match='is empty'):
            fn(imgs, m, layout, rois=[[[5, 5, 5, 9]], []])
        with pytest.raises(ValueError, match='is empty'):
            fn(imgs, m, layout, rois=[[], [[5, 5, 9, 5]]])
        with pytest.raises(ValueError, match='is empty'):
            fn(imgs, m, layout, rois=[[5, 5, 9, 5]])                         # one list of boxes for every image
        with pytest.raises(TypeError, match='UVLayout'):
            fn(imgs, m, None, rois=roi)
        with pytest.raises(ValueError, match='the UV layout has 300 vertices'):
            fn(imgs, m, UVLayout(*synthetic.make_uv_layout(3, nver=300)), rois=roi)
        with pytest.raises(IndexError, match='of UV map 1'):
            fn(imgs, [m, m[:100]], layout, rois=roi)
        if 'overlay' in name:
            with pytest.raises(ValueError, match='4-channel'):
                fn(imgs, synthetic.make_uv_map(256, 256, channels=4), layout, rois=roi)
        else:                                                                 # a 4-channel map passes the checks
            with pytest.raises(AssertionError, match='CUDA reached'):
                fn(imgs, synthetic.make_uv_map(256, 256, channels=4), layout, rois=roi)
