"""CPU checks of the image-list overlay (``syn_render_images_plan`` / ``syn_rasterize_images``, ``Sim3DR.render_images``,
``render.render_images``) without a GPU: every argument check of the two C entries fails with its own code before any
CUDA work, and the Python entries refuse mismatched lists and bad images before they touch CUDA."""
import ctypes as C

import numpy as np
import pytest

from synergynet_b200 import _lib


def _fails(code, want, text):
    assert code == want, (code, _lib.load().syn_last_error())
    assert text in _lib.load().syn_last_error(), _lib.load().syn_last_error()


# three images of 4x5, 2x3 and 1x1 pixels, packed back to back: 60 + 18 + 3 bytes
TABLE = [[0, 4, 5], [60, 2, 3], [78, 1, 1]]
BYTES = 81


def _table(rows):
    return np.ascontiguousarray(np.array(rows, np.int64).reshape(-1, 3))


def test_image_entries_reject_bad_arguments():
    lib = _lib.load()
    p = C.c_void_p(8)                                      # never dereferenced: every call below fails validation first
    start = np.array([0, 2, 2, 5], np.int32)
    good = _table(TABLE)

    def plan(v=p, m=5, nver=10, tri=p, ntri=4, st=start, std=p, tb=good, tbd=p, n=3, nbytes=BYTES, c=3, boxes=p, off=p, sv=1):
        return lib.syn_render_images_plan(v, 30, sv, 10, m, nver, tri, ntri, None if st is None else st.ctypes.data, std,
                                          None if tb is None else tb.ctypes.data, tbd, n, nbytes, c, boxes, off, None)

    _fails(plan(v=None), 1, b'syn_render_images_plan: null pointer')
    _fails(plan(st=None), 1, b'null pointer')
    _fails(plan(std=None), 1, b'null pointer')
    _fails(plan(tb=None), 1, b'null pointer')
    _fails(plan(tbd=None), 1, b'null pointer')
    _fails(plan(tri=None), 1, b'null pointer or negative triangle count')
    _fails(plan(boxes=None), 1, b'null pointer')
    _fails(plan(off=None), 1, b'null pointer')
    _fails(plan(m=0), 1, b'no mesh')
    _fails(plan(sv=0), 1, b'non-positive stride')
    _fails(plan(n=0), 1, b'0 images')
    big = np.array([0, 70000], np.int32)
    _fails(plan(m=70000, st=big, n=1, tb=_table(TABLE[:1])), 1, b'1..65535')
    many = np.zeros(65537, np.int32)
    many[-1] = 5
    _fails(plan(st=many, n=65536), 1, b'65536 images')
    # mesh_start: not from 0, not to n_meshes, not monotone
    for bad, text in (([1, 2, 2, 5], b'must run from 0 to 5'), ([0, 2, 2, 4], b'must run from 0 to 5'),
                      ([0, 3, 2, 5], b'not monotone at image 1 (2 after 3)')):
        _fails(plan(st=np.array(bad, np.int32)), 4, text)
    # the image table: out of order, overlapping, outside the bytes, empty images, offsets off the pixel grid
    for rows, nbytes, text in (
            ([[0, 4, 5], [78, 1, 1], [60, 2, 3]], BYTES, b'image 2 (2x3 at byte 60) does not fit'),       # out of order
            ([[0, 4, 5], [57, 2, 3], [78, 1, 1]], BYTES, b'image 1 (2x3 at byte 57) does not fit'),       # overlaps image 0
            ([[0, 4, 5], [60, 2, 3], [78, 1, 1]], 80, b'image 2 (1x1 at byte 78) does not fit the 80 image bytes'),
            ([[0, 4, 5], [60, 2, 3], [81, 1, 1]], BYTES, b'image 2 (1x1 at byte 81) does not fit'),       # past the end
            ([[-3, 4, 5], [60, 2, 3], [78, 1, 1]], BYTES, b'image 0 (4x5 at byte -3) does not fit'),
            ([[0, 4, 5], [60, 0, 3], [78, 1, 1]], BYTES, b'image 1 is 0x3'),
            ([[0, 4, 5], [60, 2, -1], [78, 1, 1]], BYTES, b'image 1 is 2x-1'),
            ([[0, 4, 5], [60, 2, 3], [79, 1, 1]], 83, b'image 2 starts at byte 79, not a multiple of its 3 channels')):
        _fails(plan(tb=_table(rows), nbytes=nbytes), 4, text)
    _fails(plan(c=0), 4, b'0 image channels')
    _fails(plan(nbytes=-1), 4, b'-1 image bytes')
    # a gap between two images is allowed by the table check; it then fails only on the null pointers below
    _fails(plan(tb=_table([[0, 4, 5], [63, 2, 3], [81, 1, 1]]), nbytes=84, tri=None), 1, b'null pointer or negative triangle count')

    def rast(im=p, sol=p, nbytes=BYTES, tb=good, tbd=p, n=3, c=3, cc=3, st=start, std=p, boxes=p, off=p, nkeys=100, keys=p, ws=100,
             m=5, ntri=4):
        return lib.syn_rasterize_images(im, sol, nbytes, None if tb is None else tb.ctypes.data, tbd, n, c, p, 30, 1, 10, m, 10, p, ntri, p,
                                        cc, None if st is None else st.ctypes.data, std, boxes, off, nkeys, keys, ws, None)

    _fails(rast(im=None), 1, b'syn_rasterize_images: null pointer')
    for kw in ('sol', 'tb', 'tbd', 'st', 'std', 'boxes', 'off', 'keys'):
        _fails(rast(**{kw: None}), 1, b'null pointer')
    _fails(rast(ntri=-1), 1, b'negative triangle count')
    _fails(rast(cc=4), 4, b'3 image channels, colours of 4 channels')
    _fails(rast(c=4, cc=4), 4, b'does not fit')                            # 4-channel images do not fit 81 bytes
    _fails(rast(ws=99), 4, b'key workspace of 99 slots, the plan needs 100')
    _fails(rast(nkeys=-1), 4, b'key workspace')
    _fails(rast(st=np.array([0, 4, 2, 5], np.int32)), 4, b'not monotone at image 1')
    _fails(rast(tb=_table([[0, 4, 5], [60, 2, 3], [78, 2, 1]])), 4, b'image 2 (2x1 at byte 78) does not fit')
    _fails(rast(n=0), 1, b'0 images')


def test_render_images_refuses_bad_lists_before_cuda():
    """Every refusal here comes before the CUDA check, so it is the same ValueError with or without a GPU."""
    from synergynet_b200 import Sim3DR, render
    images = [np.zeros((4, 5, 3), np.uint8), np.zeros((2, 7, 3), np.uint8)]
    tri = np.zeros((1, 3), np.int32)
    with pytest.raises(ValueError, match='1 mesh lists and no paths for 2 images'):
        Sim3DR.render_images(images, [[]], tri)
    with pytest.raises(ValueError, match='3 paths for 2 images'):
        Sim3DR.render_images(images, [[], []], tri, wfps=['a.png', None, None])
    with pytest.raises(ValueError, match='every image must be'):
        Sim3DR.render_images([images[0], np.zeros((2, 7, 4), np.uint8)], [[], []], tri)
    with pytest.raises(ValueError, match='every image must be'):
        Sim3DR.render_images([np.zeros((0, 7, 3), np.uint8)], [[]], tri)
    with pytest.raises(ValueError, match='no images'):
        Sim3DR.render_images([], [], tri)
    with pytest.raises(ValueError, match='3 mesh lists'):
        render.render_images(images, [[], [], []], connectivity=tri.T)
