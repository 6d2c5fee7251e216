"""Host side of the image-list path (no device): argument checks of the ragged C entries, the packing offsets, per-image
prior counts and shrink sizes, the ragged crop plan's tables, and chunking at SYN_FB_MAX_FRAMES images."""
import numpy as np
import pytest
import torch

from synergynet_b200 import _lib, detect, faceboxes, inference


def _fails(code, text, want=1):
    assert code == want, (code, _lib.load().syn_last_error())
    assert text in _lib.load().syn_last_error(), _lib.load().syn_last_error()


def _i32(*v):
    return np.ascontiguousarray(v, dtype=np.int32)


def test_network_and_decode_entries_reject_bad_arguments():
    lib = _lib.load()
    buf = np.zeros(64, np.int32)
    p = buf.ctypes.data                      # a non-null address; every call below fails before anything reads it
    hs, ws = _i32(64, 32), _i32(48, 1)
    _fails(lib.syn_fb_forward_images(None, p, 2, hs.ctypes.data, ws.ctypes.data, p, p, None), b'syn_fb_forward_images: bad argument')
    _fails(lib.syn_fb_forward_images(None, p, 0, hs.ctypes.data, ws.ctypes.data, p, p, None), b'0 images')
    _fails(lib.syn_fb_forward_images(None, p, 2, None, ws.ctypes.data, p, p, None), b'bad argument')
    _fails(lib.syn_fb_forward_images(None, p, 65, hs.ctypes.data, ws.ctypes.data, p, p, None), b'65 frames, 1..64 per call')
    _fails(lib.syn_fb_debug_forward_images_until(p, p, 65, hs.ctypes.data, ws.ctypes.data, 5, p, 8, p, p, None), b'65 frames, 1..64')
    _fails(lib.syn_fb_debug_forward_images_until(None, p, 2, hs.ctypes.data, ws.ctypes.data, 5, p, 8, p, p, None), b'null handle or output')
    _fails(lib.syn_fb_debug_forward_images_until(None, p, 0, hs.ctypes.data, ws.ctypes.data, 5, p, 8, p, p, None), b'null handle or output')
    for stage in (-1, 39):
        _fails(lib.syn_fb_debug_forward_images_until(None, p, 2, hs.ctypes.data, ws.ctypes.data, stage, p, 8, p, p, None), b'outside 0..38')
    sc = np.ascontiguousarray([1.0, 0.5], np.float32)
    dec = lambda n, h, w, s, k=10, loc=p: lib.syn_faceboxes_decode_images(loc, p, n, h.ctypes.data, w.ctypes.data, s.ctypes.data, 0.05,
                                                                          k, p, p, p, None)
    _fails(dec(2, hs, ws, sc, loc=None), b'null pointer')
    _fails(dec(2, hs, ws, sc, k=0), b'top_k < 1')
    _fails(dec(0, hs, ws, sc), b'0 images')
    _fails(dec(_lib.FB_MAX_FRAMES + 1, hs, ws, sc), b'1..64 per call')
    _fails(dec(2, _i32(64, 0), ws, sc), b'image 1 is 0x1')
    _fails(dec(2, hs, ws, np.ascontiguousarray([1.0, 0.0], np.float32)), b'image 1 is 32x1 at scale 0')


def test_crop_entries_reject_bad_arguments():
    lib = _lib.load()
    buf = np.zeros(4096, np.uint8)
    p = buf.ctypes.data
    rois = _i32(0, 0, 20, 20, -5, -5, 30, 30)
    idx, hs, ws, oh, ow = _i32(0, 1), _i32(64, 32), _i32(48, 40), _i32(8, 12), _i32(8, 6)
    n = int(lib.syn_crop_resize_images_plan_size(2, oh.ctypes.data, ow.ctypes.data, inference.INTER_LINEAR))
    assert n == 2 * 40 + int(lib.syn_crop_resize_plan_size(1, 8, 8, 1)) + int(lib.syn_crop_resize_plan_size(1, 12, 6, 1))
    assert lib.syn_crop_resize_images_plan_size(2, oh.ctypes.data, _i32(8, 0).ctypes.data, 1) == -1
    assert lib.syn_crop_resize_images_plan_size(2, oh.ctypes.data, ow.ctypes.data, 3) == -1

    def plan(rois=rois, idx=idx, nim=2, hs=hs, ws=ws, oh=oh, ow=ow, mode=1, nbytes=n):
        return lib.syn_crop_resize_plan_images_host(rois.ctypes.data, idx.ctypes.data if idx is not None else None, nim, hs.ctypes.data,
                                                    ws.ctypes.data, 2, oh.ctypes.data, ow.ctypes.data, mode, p, nbytes)
    _fails(plan(idx=None), b'null pointer or empty batch')
    _fails(plan(nim=0), b'0 images')
    _fails(plan(mode=3), b'interpolation 3', want=6)
    _fails(plan(hs=_i32(64, 0)), b'image 1 is 0x40')
    _fails(plan(ow=_i32(8, 0)), b'ROI 1 output 12x0')
    _fails(plan(rois=_i32(0, 0, 20, 20, 5, 5, 5, 30)), b'ROI 1 (5,5,5,30) is empty', want=4)
    _fails(plan(idx=_i32(0, 2)), b'ROI 1 names image 2 of 2', want=4)
    _fails(plan(nbytes=n - 1), b'needed', want=4)
    assert plan() == 0

    def launch(img=p, batch=2, oh=oh, ow=ow, mode=1, planar=1):
        return lib.syn_crop_resize_images(img, p, batch, oh.ctypes.data, ow.ctypes.data, mode, planar, p, None)
    _fails(launch(img=None), b'syn_crop_resize_images: null pointer')
    _fails(launch(batch=0), b'empty batch')
    _fails(launch(mode=2), b'interpolation 2', want=6)
    _fails(launch(planar=2), b'planar = 2')
    _fails(launch(oh=_i32(-1, 12)), b'ROI 0 output -1x8')
    _fails(launch(batch=70000), b'70000 ROIs', want=4)


def test_ragged_plan_holds_the_one_image_tables():
    """Each ROI's slice of a ragged plan is, byte for byte, the one-image plan of that ROI alone; the header names its
    image's bytes, size, output size and output offset."""
    lib = _lib.load()
    sizes = [(64, 48), (1, 1), (300, 17)]
    rois = [[0, 0, 20, 20], [-5, -5, 30, 30], [3, -9, 17, 280], [-1, 0, 1, 1]]
    img = [0, 2, 2, 1]
    dsz = [(8, 8), (120, 120), (7, 33), (5, 2)]
    for mode in (inference.INTER_LINEAR, inference.INTER_LANCZOS4):
        oh, ow = _i32(*[d[1] for d in dsz]), _i32(*[d[0] for d in dsz])
        n = int(lib.syn_crop_resize_images_plan_size(4, oh.ctypes.data, ow.ctypes.data, mode))
        plan = np.zeros(n, np.uint8)
        hs, ws = _i32(*[s[0] for s in sizes]), _i32(*[s[1] for s in sizes])
        r = np.ascontiguousarray(rois, np.int32)
        _lib.check(lib.syn_crop_resize_plan_images_host(r.ctypes.data, _i32(*img).ctypes.data, 3, hs.ctypes.data, ws.ctypes.data, 4,
                                                        oh.ctypes.data, ow.ctypes.data, mode, plan.ctypes.data, n))
        hdr = np.frombuffer(plan[:160].tobytes(), dtype=np.dtype([('src', '<i8'), ('h', '<i4'), ('w', '<i4'), ('oh', '<i4'),
                                                                  ('ow', '<i4'), ('out', '<i8'), ('plan', '<i8')]))
        src = [0, 3 * 64 * 48, 3 * 64 * 48 + 3]
        out = 0
        for b in range(4):
            one = inference.resize_plan(np.array([rois[b]], np.int32), dsz[b][1], dsz[b][0], mode)
            at = int(hdr['plan'][b])
            assert np.array_equal(plan[at:at + one.size], one), (mode, b)
            assert (int(hdr['src'][b]), int(hdr['h'][b]), int(hdr['w'][b])) == (src[img[b]],) + sizes[img[b]]
            assert (int(hdr['oh'][b]), int(hdr['ow'][b]), int(hdr['out'][b])) == (dsz[b][1], dsz[b][0], out)
            out += 3 * dsz[b][0] * dsz[b][1]
        assert int(hdr['plan'][3]) + inference.resize_plan(np.array([rois[3]], np.int32), 2, 5, mode).size == n


def test_packing_offsets_and_prior_counts():
    sizes = [(1, 1), (1, 333), (720, 1080), (250, 333), (1, 1)]
    rng = np.random.default_rng(0)
    host = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    pack = inference.pack_images(host, 'cpu')
    assert pack.sizes == sizes and len(pack) == 5
    assert pack.offsets == [0, 3, 3 + 999, 3 + 999 + 3 * 720 * 1080, 3 + 999 + 3 * 720 * 1080 + 3 * 250 * 333,
                            3 + 999 + 3 * 720 * 1080 + 3 * 250 * 333 + 3]
    for i in range(5):
        assert np.array_equal(pack.image(i).numpy(), host[i])
    sub = pack.slice(2, 4)
    assert sub.sizes == sizes[2:4] and np.array_equal(sub.image(1).numpy(), host[3])
    hs, ws = pack.arrays()
    assert hs.dtype == np.int32 and hs.tolist() == [s[0] for s in sizes] and ws.tolist() == [s[1] for s in sizes]
    assert inference.pack_images(pack, 'cpu') is pack
    # P_i: prior_box.py's three levels of ceil(size / step) cells (21 anchors on the first)
    c = lambda n, s: -(-n // s)
    for h, w in sizes + [(33, 993), (1079, 1023)]:
        assert detect.num_priors(h, w) == 21 * c(h, 32) * c(w, 32) + c(h, 64) * c(w, 64) + c(h, 128) * c(w, 128)
    with pytest.raises(ValueError, match='at least one image'):
        inference.pack_images([], 'cpu')
    with pytest.raises(ValueError, match=r'\(H,W,3\)'):
        inference.pack_images([np.zeros((4, 4), np.uint8)], 'cpu')
    with pytest.raises(ValueError, match='uint8'):
        inference.pack_images([torch.zeros((4, 4, 3))], 'cpu')
    with pytest.raises(ValueError, match='bytes for images of'):
        inference.ImagePack(torch.zeros(10, dtype=torch.uint8), [(2, 2)])


@pytest.mark.parametrize('hw,want', [
    ((720, 1080), (1, (1080, 720))),            # fits: no shrink
    ((719, 1080), (1, (1080, 719))),
    ((1440, 1080), (0.5, (540, 720))),          # 720 / 1440; the width then fits
    ((500, 4000), (0.27, (1080, 135))),         # only the width: 1080 / 4000
    ((1080, 1920), (0.5625, (1080, 607))),      # 2/3, then 1080 / 1280: 1920 * 0.5625 = 1080, 1080 * 0.5625 = 607.5
    ((1500, 900), (0.48, (432, 720))),          # 720 / 1500; 900 * 0.48 = 432
    ((2160, 3840), (0.28125, (1080, 607))),     # 1/3, then 1080 / 1280
])
def test_shrink_sizes(hw, want):
    """FaceBoxes/FaceBoxes.py:62-79 worked by hand: scale = 720 / h above 720 rows, then times 1080 / (w * scale) if still
    wider than 1080; cv2.resize's dsize = (int(scale * w), int(scale * h)).  __call__, detect_batch and detect_images all
    take their shrink from shrink_size, and the GPU tests hold detect_images to __call__."""
    h, w = hw
    scale, dsize = faceboxes.shrink_size(h, w)
    assert dsize == want[1] and scale == pytest.approx(want[0], rel=1e-15, abs=0)
    assert (scale == 1) == (h <= 720 and w <= 1080)


def test_pack_on_another_device_is_moved():
    pack = inference.pack_images([np.zeros((2, 3, 3), np.uint8), np.ones((1, 1, 3), np.uint8)], 'cpu')
    assert inference.pack_images(pack, 'cpu') is pack
    moved = inference.pack_images(pack, 'meta')
    assert moved.data.device.type == 'meta' and moved.sizes == pack.sizes and moved.offsets == pack.offsets


def test_chunks_of_64_images():
    assert inference.chunk_ranges(1, _lib.FB_MAX_FRAMES) == [(0, 1)]
    assert inference.chunk_ranges(64, _lib.FB_MAX_FRAMES) == [(0, 64)]
    assert inference.chunk_ranges(65, _lib.FB_MAX_FRAMES) == [(0, 64), (64, 65)]
    assert inference.chunk_ranges(130, _lib.FB_MAX_FRAMES) == [(0, 64), (64, 128), (128, 130)]
