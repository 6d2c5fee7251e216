"""Host side of the frame-batch path (no device): argument checks of the batched C entries, and the pure-Python
bookkeeping that stacks frames, splits a stack into chunks and hands the faces back to their frames."""
import numpy as np
import pytest

from synergynet_b200 import _lib, inference


def _fails(code, text):
    assert code == 1, code
    assert text in _lib.load().syn_last_error(), _lib.load().syn_last_error()


def test_batch_entries_reject_null_handles_and_bad_arguments():
    lib = _lib.load()
    buf = np.zeros(64, np.int32)
    p = buf.ctypes.data                      # a non-null address; every call below fails before anything reads it
    _fails(lib.syn_fb_forward_batch(None, p, 2, 64, 64, p, p, None), b'syn_fb_forward_batch: bad argument')
    _fails(lib.syn_fb_forward_batch(None, p, 0, 64, 64, p, p, None), b'syn_fb_forward_batch: 0 frames')
    _fails(lib.syn_fb_forward_batch(None, p, -3, 64, 64, p, p, None), b'-3 frames')
    _fails(lib.syn_fb_debug_forward_batch_until(None, p, 2, 64, 64, 5, p, 8, p, p, None), b'null handle or output')
    for stage in (-1, 39):
        _fails(lib.syn_fb_debug_forward_batch_until(None, p, 2, 64, 64, stage, p, 8, p, p, None), b'outside 0..38')
    _fails(lib.syn_faceboxes_decode_batch(None, p, 2, 64, 64, 64.0, 64.0, 1.0, 0.05, 10, p, p, p, None), b'syn_faceboxes_decode_batch: bad argument')
    _fails(lib.syn_faceboxes_decode_batch(p, p, 0, 64, 64, 64.0, 64.0, 1.0, 0.05, 10, p, p, p, None), b'syn_faceboxes_decode_batch: bad argument')
    _fails(lib.syn_faceboxes_decode_batch(p, p, 2, 64, 64, 64.0, 64.0, 0.0, 0.05, 10, p, p, p, None), b'syn_faceboxes_decode_batch: bad argument')
    _fails(lib.syn_faceboxes_decode_batch(p, p, _lib.FB_MAX_FRAMES + 1, 64, 64, 64.0, 64.0, 1.0, 0.05, 10, p, p, p, None), b'at most 64')
    _fails(lib.syn_nms_batch(None, p, 2, 10, 0.3, 0, p, p, p, None), b'syn_nms_batch: null pointer')
    _fails(lib.syn_nms_batch(p, None, 2, 10, 0.3, 0, p, p, p, None), b'syn_nms_batch: null pointer')
    _fails(lib.syn_nms_batch(p, p, 0, 10, 0.3, 0, p, p, p, None), b'no frame or no row')
    _fails(lib.syn_nms_batch(p, p, 2, 0, 0.3, 0, p, p, p, None), b'no frame or no row')
    _fails(lib.syn_nms_batch(p, p, 2, 10, 0.3, 7, p, p, p, None), b'unknown mode 7')
    _fails(lib.syn_nms_batch(p, p, _lib.FB_MAX_FRAMES + 1, 10, 0.3, 0, p, p, p, None), b'at most 64')
    _fails(lib.syn_crop_resize_batch(None, 2, 64, 64, 3, p, 1, 8, 8, 1, p, 192, 8, 1, 64, None), b'syn_crop_resize_batch: null pointer')
    _fails(lib.syn_crop_resize_batch(p, 0, 64, 64, 3, p, 1, 8, 8, 1, p, 192, 8, 1, 64, None), b'syn_crop_resize_batch: 0 frames')
    _fails(lib.syn_crop_resize_batch(p, 2, 64, 64, 3, p, 0, 8, 8, 1, p, 192, 8, 1, 64, None), b'empty batch')
    assert lib.syn_crop_resize_batch(p, 2, 64, 64, 4, p, 1, 8, 8, 1, p, 192, 8, 1, 64, None) == 6          # SYN_ERR_UNSUPPORTED


def test_frame_plan_builder_checks_the_frame_indices():
    lib = _lib.load()
    rois = np.array([[0, 0, 20, 20], [-5, -5, 30, 30]], np.int32)
    n = int(lib.syn_crop_resize_plan_size(2, 8, 8, inference.INTER_LINEAR))
    plan = np.zeros(n, np.uint8)
    args = lambda fr, nf: (rois.ctypes.data, fr.ctypes.data if fr is not None else None, nf, 2, 8, 8, inference.INTER_LINEAR,
                           plan.ctypes.data, n)
    _fails(lib.syn_crop_resize_plan_frames_host(*args(None, 3)), b'null frame list')
    _fails(lib.syn_crop_resize_plan_frames_host(*args(np.array([0, 1], np.int32), 0)), b'no frame')
    for bad in ([0, 3], [-1, 0]):
        assert lib.syn_crop_resize_plan_frames_host(*args(np.array(bad, np.int32), 3)) == 4                 # SYN_ERR_SHAPE
        assert b'names frame' in lib.syn_last_error()
    # the tables of a frame plan are those of the one-image plan: only the header's frame index differs
    one = inference.resize_plan(rois, 8, 8, inference.INTER_LANCZOS4)
    many = inference.resize_plan(rois, 8, 8, inference.INTER_LANCZOS4, [2, 0], 3)
    hdr = np.frombuffer(many[:64].tobytes(), np.int32).reshape(2, 8)
    assert hdr[:, 5].tolist() == [2, 0] and np.frombuffer(one[:64].tobytes(), np.int32).reshape(2, 8)[:, 5].tolist() == [0, 0]
    assert np.array_equal(one[64:], many[64:]) and np.array_equal(np.delete(hdr, 5, 1), np.delete(np.frombuffer(one[:64].tobytes(), np.int32).reshape(2, 8), 5, 1))
    with pytest.raises(ValueError, match='1 frame indices for 2 ROIs'):
        inference.resize_plan(rois, 8, 8, inference.INTER_LINEAR, [0], 3)


@pytest.mark.parametrize('counts', [[0, 3, 2], [3, 2, 0], [3, 0, 0, 2, 1], [0, 0, 0], [0, 5, 0], [4]])
def test_faces_return_to_their_frames(counts):
    """Empty frames first, last and in the middle: every face goes back to its frame, in order."""
    faces = [f'face{i}' for i in range(sum(counts))]
    per_frame = inference.split_by_counts(faces, counts)
    assert [len(p) for p in per_frame] == counts
    assert [f for p in per_frame for f in p] == faces
    arr = np.arange(sum(counts) * 6).reshape(sum(counts), 3, 2)                     # ndarray rows (landmarks) split the same way
    got = inference.split_by_counts(arr, counts)
    assert [len(p) for p in got] == counts and all(np.array_equal(a, arr[i]) for i, a in enumerate(x for p in got for x in p))


def test_split_rejects_counts_that_do_not_add_up():
    with pytest.raises(ValueError, match='5 items for counts that sum to 4'):
        inference.split_by_counts(list(range(5)), [1, 3])


@pytest.mark.parametrize('n', [1, 63, 64, 65, 128, 200])
def test_chunks_visit_every_frame_once_in_order(n):
    chunks = inference.chunk_ranges(n, _lib.FB_MAX_FRAMES)
    assert [i for a, b in chunks for i in range(a, b)] == list(range(n))
    assert all(0 < b - a <= _lib.FB_MAX_FRAMES for a, b in chunks) and len(chunks) == -(-n // _lib.FB_MAX_FRAMES)
    assert inference.chunk_ranges(0, 4) == []
    with pytest.raises(ValueError):
        inference.chunk_ranges(3, 0)


def test_frame_limit_is_the_headers():
    import re
    text = open(_lib.HEADER_PATH).read()
    assert int(re.search(r'#define SYN_FB_MAX_FRAMES (\d+)', text).group(1)) == _lib.FB_MAX_FRAMES


def test_stacking_frames_on_the_host():
    a, b = np.full((4, 5, 3), 7, np.uint8), np.full((4, 5, 3), 9, np.uint8)
    st = inference.stack_frames_host([a, b])
    assert st.shape == (2, 4, 5, 3) and st.dtype == np.uint8 and st.flags.c_contiguous and st[1, 0, 0, 0] == 9
    assert inference.stack_frames_host(st) is st or np.array_equal(inference.stack_frames_host(st), st)
    with pytest.raises(ValueError, match='4x5x3, 4x6x3'):
        inference.stack_frames_host([a, np.zeros((4, 6, 3), np.uint8)])
    with pytest.raises(ValueError, match='no frames'):
        inference.stack_frames_host([])
    with pytest.raises(ValueError, match=r'\(N,H,W,3\)'):
        inference.stack_frames_host(np.zeros((2, 4, 5, 4), np.uint8))
