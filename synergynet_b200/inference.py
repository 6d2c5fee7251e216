"""Host-side API semantics around the hot path, batched (reference ``utils/inference.py``).

Only tiny per-face affine algebra, the integer ROI crop (the host restatement the tests compare against) and its
device twin ``crop_resize_device`` live here; vertex reconstruction and the pose decode run on the GPU
(``Engine.reconstruct``, ``Engine.pose_decode``).
"""
from __future__ import annotations

import ctypes as C
import math
import threading
from math import cos, sin
from typing import Optional, Sequence, Tuple

import numpy as np

STD_SIZE = 120
INTER_LINEAR, INTER_LANCZOS4 = 1, 4        # cv2's constants, for crop_resize_device


def parse_param(param: np.ndarray):
    """Slices of one de-whitened 62-vector (utils/inference.py:25-31)."""
    cam = param[:12].reshape(3, 4)
    return cam[:, :3], cam[:, 3:4], param[12:52].reshape(40, 1), param[52:62].reshape(10, 1)


def roi_ints(roi_box: Sequence[float]) -> list:
    """``x0, y0, x1, y1`` of a crop: ``int(round(v))`` with Python's round-half-even (utils/inference.py:98)."""
    return [int(round(v)) for v in roi_box[:4]]


def crop_img(img: np.ndarray, roi_box: Sequence[float]) -> np.ndarray:
    """Integer-rounded ROI crop with zero fill outside the image (utils/inference.py:95-125).
    Index arithmetic is bit-exact with the reference: Python ``round`` then clamping."""
    img_h, img_w = img.shape[:2]
    x0, y0, x1, y1 = roi_ints(roi_box)
    out = np.zeros((y1 - y0, x1 - x0) + tuple(img.shape[2:]), dtype=np.uint8)
    src_x0, src_y0 = max(x0, 0), max(y0, 0)
    src_x1, src_y1 = min(x1, img_w), min(y1, img_h)
    dst_x0, dst_y0 = src_x0 - x0, src_y0 - y0
    dst_x1 = (x1 - x0) - (x1 - src_x1)
    dst_y1 = (y1 - y0) - (y1 - src_y1)
    out[dst_y0:dst_y1, dst_x0:dst_x1] = img[src_y0:src_y1, src_x0:src_x1]
    return out


def resize_plan(rois: np.ndarray, out_h: int, out_w: int, interpolation: int, frame_index=None, n_frames: int = 0) -> np.ndarray:
    """Host-built tap tables for ``crop_resize_device`` (``syn_crop_resize_plan_host``): ``rois`` (B,4) int32 x0, y0, x1, y1.
    With ``frame_index`` (B,), the plan of ``crop_resize_frames_device``: ROI b reads frame ``frame_index[b]`` of ``n_frames``."""
    from . import _lib
    lib = _lib.load()
    rois = np.ascontiguousarray(rois, dtype=np.int32).reshape(-1, 4)
    n = int(lib.syn_crop_resize_plan_size(rois.shape[0], out_h, out_w, interpolation))
    plan = np.zeros(max(n, 1), np.uint8)
    if frame_index is None:
        _lib.check(lib.syn_crop_resize_plan_host(rois.ctypes.data, rois.shape[0], out_h, out_w, interpolation, plan.ctypes.data, n))
    else:
        fi = np.ascontiguousarray(frame_index, dtype=np.int32).reshape(-1)
        if fi.shape[0] != rois.shape[0]:
            raise ValueError(f'{fi.shape[0]} frame indices for {rois.shape[0]} ROIs')
        _lib.check(lib.syn_crop_resize_plan_frames_host(rois.ctypes.data, fi.ctypes.data, int(n_frames), rois.shape[0], out_h, out_w,
                                                        interpolation, plan.ctypes.data, n))
    return plan


def crop_resize_device(image, roi_boxes: Sequence[Sequence[float]], dsize: Tuple[int, int] = (STD_SIZE, STD_SIZE),
                       interpolation: int = INTER_LINEAR, planar: bool = True):
    """Device twin of ``cv2.resize(crop_img(img, box), dsize, interpolation=...)`` for every box, byte for byte.

    ``image``: (H,W,3) uint8 BGR CUDA tensor; ``dsize`` = (width, height) as cv2 takes it; ``interpolation``:
    ``INTER_LINEAR`` or ``INTER_LANCZOS4``.  Returns uint8 (B,3,h,w) crops when ``planar`` (the backbone's input layout,
    ``permute(0,3,1,2)`` of the stacked crops), else (B,h,w,3).  Runs on the current stream of the image's device."""
    import torch
    from . import _lib
    if image.dtype != torch.uint8 or image.dim() != 3 or not image.is_cuda or not image.is_contiguous():
        raise ValueError('image must be a contiguous (H,W,C) uint8 CUDA tensor')
    out_w, out_h = int(dsize[0]), int(dsize[1])
    plan = torch.from_numpy(resize_plan(np.array([roi_ints(b) for b in roi_boxes], np.int32), out_h, out_w, interpolation))
    plan = plan.to(image.device)
    B = len(roi_boxes)
    if planar:
        out = torch.empty((B, 3, out_h, out_w), dtype=torch.uint8, device=image.device)
        strides = (3 * out_h * out_w, out_w, 1, out_h * out_w)
    else:
        out = torch.empty((B, out_h, out_w, 3), dtype=torch.uint8, device=image.device)
        strides = (3 * out_h * out_w, 3 * out_w, 3, 1)
    _lib.launch(image.device, 'syn_crop_resize', image.data_ptr(), image.shape[0], image.shape[1], image.shape[2], plan.data_ptr(), B,
                out_h, out_w, interpolation, out.data_ptr(), *strides)
    return out


def crop_resize_frames_device(frames, frame_index: Sequence[int], roi_boxes: Sequence[Sequence[float]],
                              dsize: Tuple[int, int] = (STD_SIZE, STD_SIZE), interpolation: int = INTER_LINEAR, planar: bool = True):
    """:func:`crop_resize_device` for a stack of frames in one launch: ``frames`` (N,H,W,3) uint8 CUDA tensor, ROI b is
    ``roi_boxes[b]`` of frame ``frame_index[b]``.  The bytes are those of ``crop_resize_device(frames[i], ...)`` frame
    by frame; a frame may contribute any number of ROIs, none included."""
    import torch
    from . import _lib
    if frames.dtype != torch.uint8 or frames.dim() != 4 or not frames.is_cuda or not frames.is_contiguous():
        raise ValueError('frames must be a contiguous (N,H,W,C) uint8 CUDA tensor')
    out_w, out_h = int(dsize[0]), int(dsize[1])
    B = len(roi_boxes)
    plan = torch.from_numpy(resize_plan(np.array([roi_ints(b) for b in roi_boxes], np.int32), out_h, out_w, interpolation,
                                        frame_index, int(frames.shape[0]))).to(frames.device)
    if planar:
        out = torch.empty((B, 3, out_h, out_w), dtype=torch.uint8, device=frames.device)
        strides = (3 * out_h * out_w, out_w, 1, out_h * out_w)
    else:
        out = torch.empty((B, out_h, out_w, 3), dtype=torch.uint8, device=frames.device)
        strides = (3 * out_h * out_w, 3 * out_w, 3, 1)
    _lib.launch(frames.device, 'syn_crop_resize_batch', frames.data_ptr(), frames.shape[0], frames.shape[1], frames.shape[2],
                frames.shape[3], plan.data_ptr(), B, out_h, out_w, interpolation, out.data_ptr(), *strides)
    return out


class ImagePack:
    """N uint8 BGR images of any sizes packed back to back on one device: ``data`` is a flat uint8 CUDA tensor, image i
    ((h_i, w_i, 3), ``sizes[i] = (h_i, w_i)``) starting at byte ``offsets[i]`` = sum of 3 h_j w_j over j < i -- the layout
    the ``*_images`` entries of the library take."""

    def __init__(self, data, sizes):
        self.data = data
        self.sizes = [(int(h), int(w)) for h, w in sizes]
        self.offsets = np.concatenate([[0], np.cumsum([3 * h * w for h, w in self.sizes])]).astype(np.int64).tolist()
        if int(data.numel()) != self.offsets[-1]:
            raise ValueError(f'{int(data.numel())} bytes for images of {self.offsets[-1]} bytes')

    def __len__(self):
        return len(self.sizes)

    def image(self, i: int):
        """Image i as a (h, w, 3) view."""
        h, w = self.sizes[i]
        return self.data[self.offsets[i]:self.offsets[i + 1]].view(h, w, 3)

    def slice(self, a: int, b: int) -> 'ImagePack':
        """Images a..b-1 (a view of the same bytes)."""
        return ImagePack(self.data[self.offsets[a]:self.offsets[b]], self.sizes[a:b])

    def arrays(self):
        """(heights, widths) as int32 arrays, for the C entries."""
        hw = np.array(self.sizes, np.int32).reshape(-1, 2)
        return np.ascontiguousarray(hw[:, 0]), np.ascontiguousarray(hw[:, 1])


def pack_images(images, device) -> ImagePack:
    """A list of (h_i, w_i, 3) BGR uint8 images of any sizes -> one :class:`ImagePack` on ``device``: host arrays are
    packed on the host and uploaded in one copy, CUDA tensors are packed on the device.  An ImagePack on ``device``
    passes through; one elsewhere is copied there."""
    import torch
    if isinstance(images, ImagePack):
        if images.data.device == torch.device(device):
            return images
        return ImagePack(images.data.to(device), images.sizes)                         # bytes on another device: moved
    images = list(images)
    if not images:
        raise ValueError('no images: an image list needs at least one image')
    for im in images:
        if im.ndim != 3 or im.shape[2] != 3 or im.shape[0] < 1 or im.shape[1] < 1:
            raise ValueError(f'every image must be (H,W,3) with H, W >= 1, got {tuple(im.shape)}')
        if isinstance(im, torch.Tensor) and im.dtype != torch.uint8:
            raise ValueError(f'image tensors must be uint8, got {im.dtype}')
    sizes = [(int(im.shape[0]), int(im.shape[1])) for im in images]
    if all(isinstance(im, torch.Tensor) and im.is_cuda for im in images):
        return ImagePack(torch.cat([im.to(device).reshape(-1) for im in images]), sizes)
    host = [im.cpu().numpy() if isinstance(im, torch.Tensor) else np.asarray(im) for im in images]
    flat = [np.ascontiguousarray(im, dtype=np.uint8).reshape(-1) for im in host]
    # one image is already packed: no host copy of its bytes (6 MB at 1080 x 1920) before the upload
    flat = flat[0] if len(flat) == 1 else np.concatenate(flat)
    return ImagePack(torch.from_numpy(flat).to(device), sizes)


def crop_resize_images_device(images: ImagePack, image_index: Sequence[int], roi_boxes: Sequence[Sequence[float]],
                              dsize=(STD_SIZE, STD_SIZE), interpolation: int = INTER_LINEAR, planar: bool = True):
    """:func:`crop_resize_device` for a list of images of any sizes in one launch: ROI b is ``roi_boxes[b]`` of image
    ``image_index[b]`` of the :class:`ImagePack` ``images``.  ``dsize``: one (width, height) for every ROI -- the result is
    then a (B,3,h,w) (``planar``) or (B,h,w,3) tensor -- or a list of one (width, height) per ROI, and the result is the
    flat uint8 tensor of the outputs packed back to back.  The bytes of ROI b are those of
    ``crop_resize_device(image, [roi_boxes[b]], ...)`` on its image alone."""
    import torch
    from . import _lib
    lib = _lib.load()
    B = len(roi_boxes)
    one = len(dsize) == 2 and not hasattr(dsize[0], '__len__')
    dsizes = [tuple(dsize)] * B if one else [tuple(d) for d in dsize]
    if len(dsizes) != B or len(image_index) != B:
        raise ValueError(f'{len(dsizes)} output sizes and {len(image_index)} image indices for {B} ROIs')
    out_w = np.ascontiguousarray([int(d[0]) for d in dsizes], np.int32)
    out_h = np.ascontiguousarray([int(d[1]) for d in dsizes], np.int32)
    rois = np.ascontiguousarray(np.array([roi_ints(b) for b in roi_boxes], np.int32).reshape(-1, 4))
    idx = np.ascontiguousarray(image_index, dtype=np.int32)
    hs, ws = images.arrays()
    n = int(lib.syn_crop_resize_images_plan_size(B, out_h.ctypes.data, out_w.ctypes.data, interpolation))
    plan = np.zeros(max(n, 1), np.uint8)
    _lib.check(lib.syn_crop_resize_plan_images_host(rois.ctypes.data, idx.ctypes.data, len(images), hs.ctypes.data, ws.ctypes.data, B,
                                                    out_h.ctypes.data, out_w.ctypes.data, interpolation, plan.ctypes.data, n))
    dev = images.data.device
    plan = torch.from_numpy(plan).to(dev)
    out = torch.empty((int((3 * out_h.astype(np.int64) * out_w).sum()),), dtype=torch.uint8, device=dev)
    _lib.launch(dev, 'syn_crop_resize_images', images.data.data_ptr(), plan.data_ptr(), B, out_h.ctypes.data, out_w.ctypes.data,
                interpolation, int(bool(planar)), out.data_ptr())
    if not one:
        return out
    w, h = dsizes[0]
    return out.view(B, 3, h, w) if planar else out.view(B, h, w, 3)


def stack_frames_host(frames) -> np.ndarray:
    """N equally sized (H,W,3) BGR images (a list, or one (N,H,W,3) array) -> one contiguous uint8 (N,H,W,3) array."""
    if not (isinstance(frames, np.ndarray) and frames.ndim == 4):
        frames = [np.asarray(f) for f in frames]
        if not frames:
            raise ValueError('no frames: a frame batch needs at least one image')
        shapes = [tuple(f.shape) for f in frames]
        if any(sh != shapes[0] for sh in shapes):
            sizes = ', '.join('x'.join(str(d) for d in sh) for sh in sorted(set(shapes)))
            raise ValueError(f'the frames of one batch must have one size, got {sizes}; group the frames by size, or use the '
                             '*_images methods (FaceBoxes.detect_images, get_all_outputs_images), which take images of any sizes')
        frames = np.stack(frames)
    if frames.shape[0] == 0 or frames.shape[3] != 3:
        raise ValueError(f'frames must be (N,H,W,3) with N >= 1, got {tuple(frames.shape)}')
    return np.ascontiguousarray(frames, dtype=np.uint8)


def stack_frames_device(frames, device):
    """The frame stack on ``device``: one upload of :func:`stack_frames_host`, or the (N,H,W,3) uint8 CUDA tensor the
    caller already holds (``get_all_outputs_batch`` hands its stack to the detector this way)."""
    import torch
    if isinstance(frames, torch.Tensor):
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3 or frames.shape[0] == 0:
            raise ValueError(f'a frame stack must be a uint8 (N,H,W,3) tensor with N >= 1, got {frames.dtype} {tuple(frames.shape)}')
        return frames.to(device).contiguous()
    return torch.from_numpy(stack_frames_host(frames)).to(device)


def chunk_ranges(n: int, limit: int) -> list:
    """``[(start, stop), ...]`` covering items 0..n-1 in order, at most ``limit`` each (frames per detector call, faces
    per dense reconstruction)."""
    if limit < 1:
        raise ValueError(f'chunk limit {limit}')
    return [(a, min(a + limit, n)) for a in range(0, n, limit)]


def split_by_counts(items: Sequence, counts: Sequence[int]) -> list:
    """Undo the frame -> faces flattening: ``items`` holds the faces of frame 0, then frame 1, ...; ``counts[i]`` faces
    belong to frame i (0 for a frame without a face).  Returns one list per frame."""
    if sum(counts) != len(items):
        raise ValueError(f'{len(items)} items for counts that sum to {sum(counts)}')
    out, at = [], 0
    for c in counts:
        out.append(list(items[at:at + c]))
        at += c
    return out


def square_roi(rect: Sequence[float]) -> list:
    """Enlarged square box around a detection (synergy3DMM.py:181-185): side = 1.2 x height,
    ``//`` floor division as in the reference."""
    h_center = (rect[1] + rect[3]) / 2
    w_center = (rect[0] + rect[2]) / 2
    margin = (rect[3] - rect[1]) * 1.2 // 2
    tail = list(rect[4:]) if len(rect) > 4 else [1.0]
    return [w_center - margin, h_center - margin, w_center + margin, h_center + margin] + tail


def rescale_vertices(vertex: np.ndarray, roi_box: Sequence[float]) -> np.ndarray:
    """Crop -> image coordinates for one (3,N) array (utils/inference.py:127-138)."""
    sx, sy, ex, ey = roi_box[:4]
    kx, ky = (ex - sx) / STD_SIZE, (ey - sy) / STD_SIZE
    out = np.array(vertex, copy=True)
    out[0] = out[0] * kx + sx
    out[1] = out[1] * ky + sy
    out[2] *= (kx + ky) / 2
    return out


def roi_affine(roi_boxes: Sequence[Sequence[float]]) -> np.ndarray:
    """(B,5) fp32 rows kx, sx, ky, sy, kz of the crop -> image map of ``_predict_vertices`` / ``predict_pose``
    (utils/inference.py:129-136,150-154).  The reference evaluates the scales as Python floats (double) and numpy
    rounds them to fp32 when they meet the fp32 vertex arrays; the same happens here, once per face, as index-like host
    work -- the per-vertex arithmetic runs on the GPU (``Engine.reconstruct_image``)."""
    out = np.empty((len(roi_boxes), 5), np.float32)
    for i, box in enumerate(roi_boxes):
        sx, sy, ex, ey = box[:4]
        kx, ky = (ex - sx) / STD_SIZE, (ey - sy) / STD_SIZE
        out[i] = (kx, sx, ky, sy, (kx + ky) / 2)
    return out


# lighting of the solid-mesh overlay (utils/render.py:18-27), consumed by synergynet_b200.Sim3DR.render
RENDER_CFG = {
    'intensity_ambient': 0.75, 'color_ambient': (1, 1, 1),
    'intensity_directional': 0.7, 'color_directional': (1, 1, 1),
    'intensity_specular': 0.2, 'specular_exp': 5,
    'light_pos': (0, 0, 5), 'view_pos': (0, 0, 5),
}


# ---- the pose axes (utils/inference.py:199-244, draw_axis; singleImage.py:112-117 calls it once per face) ----------------
AXIS_COLOURS = ((0, 0, 255), (0, 255, 0), (255, 0, 0))        # BGR of the x (red), y (green) and z (blue) axes
AXIS_THICKNESS = 4
_INT32 = (-2 ** 31, 2 ** 31 - 1)


def plan_axis(yaw, pitch, roll, pts68):
    """The three ``cv2.line`` segments ``draw_axis`` draws for one face: ``(segments, error)``.  ``segments`` is a list of
    ``(x0, y0, x1, y1, (b, g, r))`` integer segments, in draw order; ``error`` is None, or the exception the reference
    raises after drawing those segments (``ValueError`` for a NaN point, ``OverflowError`` for an infinite one, and
    for a point outside int32 -- where the reference's ``cv2.line`` raises ``cv2.error`` -- an ``OverflowError`` naming
    it).

    The expressions are the reference's, in its scalar types: with Python float angles and float32 ``pts68`` (what
    ``get_all_outputs`` returns), the extents' product is float32, ``size`` a Python float, and every end point
    ``size * (...) + tdx`` a NumPy float32 (NEP 50: the Python float term is cast to float32, then added), truncated
    toward zero by ``int()``.  ``math.cos`` / ``math.sin`` are libm's, as the reference's are.  ``tdx``, ``tdy`` and
    ``size`` of the reference's signature are overwritten by it, so they are not taken here."""
    try:
        pitch = pitch * np.pi / 180
        yaw = -(yaw * np.pi / 180)
        roll = roll * np.pi / 180
        tdx = pts68[0, 30]
        tdy = pts68[1, 30]
        minx, maxx = np.min(pts68[0, :]), np.max(pts68[0, :])
        miny, maxy = np.min(pts68[1, :]), np.max(pts68[1, :])
        size = math.sqrt((maxx - minx) * (maxy - miny)) * 0.5
        ends = ((size * (cos(yaw) * cos(roll)) + tdx, size * (cos(pitch) * sin(roll) + cos(roll) * sin(pitch) * sin(yaw)) + tdy),
                (size * (-cos(yaw) * sin(roll)) + tdx, size * (cos(pitch) * cos(roll) - sin(pitch) * sin(yaw) * sin(roll)) + tdy),
                (size * (sin(yaw)) + tdx, size * (-cos(yaw) * sin(pitch)) + tdy))
    except (ValueError, OverflowError) as e:             # math.cos of an infinite angle: before any line, as there
        return [], e
    segments = []
    for (x, y), colour in zip(ends, AXIS_COLOURS):
        try:
            p0, p1 = (int(tdx), int(tdy)), (int(x), int(y))
        except (ValueError, OverflowError) as e:
            return segments, e
        for p in (p0, p1):
            if not all(_INT32[0] <= v <= _INT32[1] for v in p):
                return segments, OverflowError(f'draw_axis: point {p} lies outside int32, which cv2.line cannot draw')
        segments.append((*p0, *p1, colour))
    return segments, None


def _segment_table(seg_lists, frames):
    """One int64 buffer for syn_draw_lines: frames (n,3) | seg_start (n+1) int32 | segments (S,5) int32, 8-byte aligned.
    ``frames``: (n,3) int64 byte offset, height, width.  Returns (buffer, n_segs, seg_start view, frames view)."""
    counts = [len(s) for s in seg_lists]
    n, n_segs = len(counts), sum(counts)
    start = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    segs = np.array([[x0, y0, x1, y1, b | (g << 8) | (r << 16)] for sl in seg_lists for x0, y0, x1, y1, (b, g, r) in sl],
                    np.int64).reshape(-1, 5).astype(np.int32)
    a = 3 * n
    b = a + (n + 2) // 2
    buf = np.zeros(b + (5 * n_segs + 1) // 2, np.int64)
    buf[:a] = np.asarray(frames, np.int64).reshape(-1)
    buf[a:b].view(np.int32)[:n + 1] = start
    buf[b:].view(np.int32)[:5 * n_segs] = segs.reshape(-1)
    return buf, (a, b), n_segs, start


def draw_lines_device(images, seg_lists, thickness: int = AXIS_THICKNESS):
    """``cv2.line(image, (x0, y0), (x1, y1), (b, g, r), thickness)`` for every segment of ``seg_lists[i]`` onto image i,
    in order, IN PLACE, in one launch (``syn_draw_lines``; only thickness 4 -- draw_axis's -- is restated).  ``images``:
    a contiguous uint8 (N,H,W,3) CUDA stack, or an :class:`ImagePack`.  One upload of the segments; no synchronisation."""
    import torch
    from . import _lib
    if isinstance(images, ImagePack):
        data, sizes = images.data, images.sizes
        offsets = images.offsets[:-1]
    else:
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] != 3 or not images.is_cuda or not images.is_contiguous():
            raise ValueError('images must be a contiguous uint8 (N,H,W,3) CUDA tensor or an ImagePack')
        n, h, w = (int(v) for v in images.shape[:3])
        data, sizes, offsets = images, [(h, w)] * n, [3 * h * w * i for i in range(n)]
    if len(seg_lists) != len(sizes):
        raise ValueError(f'{len(seg_lists)} segment lists for {len(sizes)} images')
    frames = np.array([[o, h, w] for o, (h, w) in zip(offsets, sizes)], np.int64)
    buf, (a, b), n_segs, start = _segment_table(seg_lists, frames)
    if n_segs == 0:
        return images
    table = torch.from_numpy(buf).to(data.device)
    _lib.launch(data.device, 'syn_draw_lines', data.data_ptr(), data.numel(), frames.ctypes.data, table.data_ptr(), len(sizes),
                start.ctypes.data, table[a:b].data_ptr(), table[b:].data_ptr(), n_segs, int(thickness), 8)
    return images


def draw_axis(img, yaw, pitch, roll, tdx=None, tdy=None, size=100, pts68=None):
    """``utils/inference.py:199-244`` on the GPU, byte for byte: the x, y and z axes of one face as three ``cv2.line``
    segments of thickness 4 from landmark 30 of ``pts68`` (3,68), scaled by the landmarks' extent; ``tdx``, ``tdy`` and
    ``size`` are ignored, as the reference overwrites them.  ``img``: a (H,W,3) uint8 BGR numpy array -- drawn on the
    device and copied back into the same array -- or a contiguous CUDA tensor, drawn in place.  Returns ``img``.

    Where the reference raises, this raises too, after drawing the axes the reference draws before the failing one: a
    NaN end point is ``ValueError``, a point outside int32 an ``OverflowError`` naming it (``cv2.error`` there)."""
    import torch
    segments, error = plan_axis(yaw, pitch, roll, pts68)
    if isinstance(img, torch.Tensor):
        if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3 or not img.is_cuda or not img.is_contiguous():
            raise ValueError('draw_axis draws on a contiguous uint8 (H,W,3) CUDA tensor or a uint8 (H,W,3) numpy array')
        if segments:
            draw_lines_device(img.unsqueeze(0), [segments])
    else:
        if not isinstance(img, np.ndarray) or img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
            raise ValueError('draw_axis draws on a contiguous uint8 (H,W,3) CUDA tensor or a uint8 (H,W,3) numpy array')
        if segments:
            if not torch.cuda.is_available():
                raise RuntimeError('draw_axis needs a CUDA device (H100, sm_90a); there is no CPU fallback')
            dev = torch.device('cuda', torch.cuda.current_device())
            canvas = torch.from_numpy(np.ascontiguousarray(img)).to(dev)
            draw_lines_device(canvas.unsqueeze(0), [segments])
            img[...] = canvas.cpu().numpy()
    if error is not None:
        raise error
    return img


# ---- OBJ text of the dense meshes (utils/inference.py:8-23 write_obj; artistic.py:19-31 write_obj_with_colors) ----------
OBJ_NEG_ZERO = -2 ** 63                 # how the C entries carry -0.0 in a '{}' field of integral floats
OBJ_CHUNK_BYTES = 1 << 30               # output text per device pass of obj_bytes (about 3.6 MB per dense face)
OBJ_MAX_MESHES = 65535                  # meshes per syn_obj_plan / syn_obj_write call


def obj_file_name(obj_name: str) -> str:
    """The file the reference writers open: ``.obj`` appended unless the last dot-separated part is ``obj``."""
    return obj_name if obj_name.split('.')[-1] == 'obj' else obj_name + '.obj'


def obj_field_values(a, what: str):
    """``(int64 array, dot0)`` of the values the reference writes with ``'{}'``: integer arrays as they are (dot0 = 0),
    float arrays whose every value is integral and below 1e16 in magnitude as their integers (dot0 = 1: printed as
    ``N.0``, -0.0 as ``-0.0``).  Any other float would need shortest-round-trip printing, which is not restated: a
    ValueError names the first one."""
    a = np.asarray(a)
    if a.dtype.kind in 'iu':
        if a.dtype.kind == 'u' and a.size and int(a.max()) > 2 ** 63 - 1:
            raise ValueError(f'{what}: {int(a.max())} does not fit int64')
        return np.ascontiguousarray(a, dtype=np.int64), 0
    if a.dtype.kind != 'f':
        raise TypeError(f'{what} must be integers or integral floats, got {a.dtype}')
    f = a.astype(np.float64)
    with np.errstate(invalid='ignore'):
        bad = ~(np.isfinite(f) & (np.floor(f) == f) & (np.abs(f) < 1e16))
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise ValueError(f'{what}{list(at)} = {f[at]!r}: only integral floats below 1e16 are written as the reference '
                         'writes them (any other float needs shortest round-trip printing)')
    out = f.astype(np.int64)
    out[(f == 0) & np.signbit(f)] = OBJ_NEG_ZERO
    return np.ascontiguousarray(out), 1


def _obj_vertices(vertices):
    """``vertices`` ((3,N) or (B,3,N) float32, numpy or CUDA) checked and seen as (B,3,N), not yet uploaded."""
    import torch
    if isinstance(vertices, torch.Tensor):
        if vertices.dtype != torch.float32:
            raise TypeError(f'vertices must be float32 (what predict_denseVert and get_all_outputs return), got {vertices.dtype}')
        if not vertices.is_cuda:
            vertices = vertices.numpy()
    if not isinstance(vertices, torch.Tensor):
        vertices = np.asarray(vertices)
        if vertices.dtype != np.float32:
            raise TypeError(f'vertices must be float32 (what predict_denseVert and get_all_outputs return), got {vertices.dtype}')
    if vertices.ndim == 2:
        vertices = vertices[None]
    if vertices.ndim != 3 or vertices.shape[1] != 3 or vertices.shape[0] < 1 or vertices.shape[2] < 1:
        raise ValueError(f'vertices must be (3,N) or (B,3,N) with B, N >= 1, got {tuple(vertices.shape)}')
    return vertices


def _obj_upload(vertices):
    """The (B,3,N) meshes of :func:`_obj_vertices` as a CUDA tensor with positive strides (host arrays: one upload)."""
    import torch
    if not isinstance(vertices, torch.Tensor):
        if not torch.cuda.is_available():
            raise RuntimeError('the OBJ encoder needs a CUDA device (H100, sm_90a); there is no CPU fallback')
        vertices = torch.from_numpy(np.ascontiguousarray(vertices)).to(torch.device('cuda', torch.cuda.current_device()))
    if min(vertices.stride()) <= 0:
        vertices = vertices.contiguous()
    return vertices


class ObjEncoder:
    """The device side of the OBJ writers on one GPU (``syn_obj_plan`` / ``syn_obj_write``) and ``launches``, the
    kernels it has launched.  It holds no device memory: every call brings its own workspace (:meth:`workspace`, 8 bytes
    per 256 lines), so calls from several host threads and streams never share one."""

    def __init__(self, device):
        import torch
        self.device = torch.device(device)
        self.launches = 0
        self._count = threading.Lock()

    def workspace(self, batch: int, n_lines: int, ntri: int):
        """A new workspace for one plan and the write that follows it."""
        import torch
        from . import _lib
        need = int(_lib.load().syn_obj_workspace_size(batch, n_lines, ntri))
        if need < 0:
            raise ValueError(f'{batch} meshes of {n_lines} vertex lines and {ntri} triangles (1..65535 meshes per call)')
        return torch.empty((need + 7) // 8, dtype=torch.int64, device=self.device)

    def _launched(self, n: int) -> None:
        with self._count:
            self.launches += n

    def plan(self, desc, ws, offsets) -> None:
        from . import _lib
        _lib.launch(self.device, 'syn_obj_plan', C.byref(desc), ws.data_ptr(), ws.numel() * 8, offsets.data_ptr())
        n_lines = desc.n_keep if desc.keep_host else desc.nver
        self._launched(2 if n_lines or desc.ntri else 1)

    def write(self, desc, ws, offsets, out) -> None:
        from . import _lib
        _lib.launch(self.device, 'syn_obj_write', C.byref(desc), ws.data_ptr(), ws.numel() * 8, offsets.data_ptr(), out.data_ptr(),
                    out.numel())
        n_lines = desc.n_keep if desc.keep_host else desc.nver
        self._launched((1 if n_lines or desc.ntri else 0) + (1 if desc.batch > 1 and desc.ntri else 0))


_obj_encoders = {}
_obj_encoders_lock = threading.Lock()


def obj_encoder(device) -> ObjEncoder:
    import torch
    device = torch.device(device)
    with _obj_encoders_lock:
        if device not in _obj_encoders:
            _obj_encoders[device] = ObjEncoder(device)
        return _obj_encoders[device]


class ObjTables:
    """The parts of an OBJ text every mesh of a call shares, checked on the host and uploaded once: the triangles (3,ntri)
    as the reference takes them, the colours -- None (write_obj's format), one (n,3) table for every mesh or (M,n,3),
    one per mesh (write_obj_with_colors' format) -- and the kept-vertex list (None: every vertex).  Every refusal
    happens here, before any CUDA call."""

    def __init__(self, triangles, nver: int, colors=None, keep=None, n_meshes: Optional[int] = None):
        tri = np.asarray(triangles)
        if tri.ndim != 2 or tri.shape[0] != 3:
            raise ValueError(f'triangles must be (3, ntri) as the reference writers take them, got {tri.shape}')
        self.tri, self.tri_dot0 = obj_field_values(tri.T, 'triangles.T')
        self.nver = int(nver)
        self.keep = None
        if keep is not None:
            k = np.asarray(keep)
            if k.ndim != 1 or k.dtype.kind not in 'iu':
                raise ValueError(f'keep must be a 1-d integer index array, got {k.dtype} {k.shape}')
            out = np.argwhere((k < 0) | (k >= self.nver))
            if out.size:
                raise ValueError(f'keep[{int(out[0, 0])}] = {int(k[out[0, 0]])} lies outside [0, {self.nver})')
            self.keep = np.ascontiguousarray(k, dtype=np.int32)
        self.n_lines = self.nver if self.keep is None else len(self.keep)
        self.colors, self.colors_dot0 = None, 0
        if colors is not None:
            col = colors.cpu().numpy() if hasattr(colors, 'cpu') else np.asarray(colors)
            if col.ndim == 2:
                col = col[None]
            if col.ndim != 3 or col.shape[1:] != (self.n_lines, 3) or (col.shape[0] != 1 and col.shape[0] != n_meshes):
                raise ValueError(f'colors must be ({self.n_lines}, 3), one row per written vertex, or one such table per mesh; got '
                                 f'{tuple(np.asarray(colors).shape)}')
            self.colors, self.colors_dot0 = obj_field_values(col, 'colors')
        self._dev = None

    def upload(self, device):
        """(triangles, keep, colours) on ``device``, one upload each, kept for the next call."""
        import torch
        if self._dev is None or self._dev[0] != device:
            up = lambda a: None if a is None else torch.from_numpy(a).to(device)
            self._dev = (device, up(self.tri), up(self.keep), up(self.colors))
        return self._dev[1:]

    def desc(self, vertices, m0: int, device, colors_dev=None):
        """The syn_obj_desc_t of the (B,3,N) device meshes ``vertices``, meshes m0.. of the call.  ``colors_dev``: the
        meshes' own (B,n,3) int64 colour rows on the device, printed as integral floats, in place of the tables' colours."""
        import torch
        from . import _lib
        tri, keep, col = self.upload(device)
        b, _, n = (int(s) for s in vertices.shape)
        if n != self.nver:
            raise ValueError(f'{n} vertices per mesh, the tables were built for {self.nver}')
        sb, sc, sv = (int(s) for s in vertices.stride())
        d = _lib.ObjDesc()
        d.vertices, d.stride_mesh, d.stride_vertex, d.stride_coord, d.batch, d.nver = vertices.data_ptr(), max(sb, 1), sv, sc, b, n
        if self.keep is not None:
            d.keep_host, d.keep_dev, d.n_keep = self.keep.ctypes.data, keep.data_ptr(), len(self.keep)
        if col is not None:
            shared = col.shape[0] == 1
            d.colors = col.data_ptr() if shared else col[m0].data_ptr()
            d.colors_stride_mesh, d.colors_dot0 = 0 if shared else 3 * self.n_lines, self.colors_dot0
        if colors_dev is not None:
            if colors_dev.dtype != torch.int64 or tuple(colors_dev.shape) != (b, self.n_lines, 3) or not colors_dev.is_contiguous() \
                    or colors_dev.device != vertices.device:
                raise ValueError(f'colors_dev must be contiguous int64 ({b}, {self.n_lines}, 3) on the meshes\' device')
            d.colors, d.colors_stride_mesh, d.colors_dot0 = colors_dev.data_ptr(), 3 * self.n_lines, 1
        d.triangles, d.ntri, d.tri_dot0 = tri.data_ptr() if tri.numel() else None, int(self.tri.shape[0]), self.tri_dot0
        d.tri_order = 0 if self.colors is None and colors_dev is None else 1
        return d

    def encode(self, vertices, m0: int = 0, chunk_bytes: int = OBJ_CHUNK_BYTES, colors_dev=None) -> list:
        """The OBJ texts of the (B,3,N) CUDA meshes ``vertices`` (meshes m0.. of the call), as a list of B ``bytes``:
        plan, one read of the offsets, write and one download per chunk of about ``chunk_bytes`` of text.  ``colors_dev``
        (B,n,3) int64 on the device: each mesh's colours, written as ``write_obj_with_colors`` writes float32 colours of
        uint8 values ("233.0")."""
        import torch
        dev = vertices.device
        enc = obj_encoder(dev)
        coloured = self.colors is not None or colors_dev is not None
        per_mesh = 40 * self.n_lines + (32 if coloured else 0) * self.n_lines + 24 * int(self.tri.shape[0]) + 1
        out = []
        for a, b in chunk_ranges(int(vertices.shape[0]), min(OBJ_MAX_MESHES, max(1, chunk_bytes // per_mesh))):
            d = self.desc(vertices[a:b], m0 + a, dev, None if colors_dev is None else colors_dev[a:b])
            ws = enc.workspace(b - a, self.n_lines, d.ntri)
            offsets = torch.empty(b - a + 1, dtype=torch.int64, device=dev)
            enc.plan(d, ws, offsets)
            off = offsets.cpu().numpy()                                   # the one host read: the size to allocate
            text = torch.empty(int(off[-1]), dtype=torch.uint8, device=dev)
            enc.write(d, ws, offsets, text)
            host = text.cpu().numpy()
            out += [host[off[i]:off[i + 1]].tobytes() for i in range(b - a)]
        return out


def obj_bytes(vertices, triangles, colors=None, keep=None) -> list:
    """The file bytes of ``write_obj(name, vertices[b], triangles)`` -- or, with ``colors``, of
    ``write_obj_with_colors(name, vertices[b][:, keep], triangles, colors)`` -- for every mesh b, encoded on the GPU: a
    list of B ``bytes``.  ``vertices``: float32 (B,3,N) or (3,N), a CUDA tensor of any strides (the dense output of
    ``reconstruct_image`` as it is) or a numpy array (uploaded once).  ``triangles`` (3,ntri), integers or integral
    floats, written as given.  ``colors``: (n,3) for every mesh or (B,n,3), BGR as stored, n the written vertex count.
    ``keep``: the kept vertex indices (``vertices[:, keep]`` without a gather copy)."""
    v = _obj_vertices(vertices)
    tables = ObjTables(triangles, int(v.shape[2]), colors, keep, int(v.shape[0]))       # every refusal before CUDA
    return tables.encode(_obj_upload(v))


def write_obj(obj_name, vertices, triangles):
    """``utils/inference.py:8-23``, the same file bytes, encoded on the GPU: one ``'v {:.4f} {:.4f} {:.4f}'`` line per
    vertex of the float32 (3,N) ``vertices`` (numpy or CUDA), one ``'f {} {} {}'`` line per triangle of (3,ntri)
    ``triangles`` in the order 2, 1, 0, to ``obj_name`` (``.obj`` appended unless it ends so)."""
    triangles = triangles.copy()
    text = obj_bytes(vertices, triangles)[0]
    with open(obj_file_name(obj_name), 'wb') as f:
        f.write(text)


def write_obj_with_colors(obj_name, vertices, triangles, colors):
    """``artistic.py:19-31`` (= ``uv_texture_realFaces.py:21-33``), the same file bytes, encoded on the GPU: each vertex
    line continues with ``colors[i, 2], [i, 1], [i, 0]`` (uint8 colours as digits, float colours from uint8 as
    ``233.0``); the triangle lines are in the order 0, 1, 2."""
    triangles = triangles.copy()
    text = obj_bytes(vertices, triangles, colors)[0]
    with open(obj_file_name(obj_name), 'wb') as f:
        f.write(text)


# ---- UV textures (artistic.py:49-53,126-131; uv_texture_realFaces.py:47-51,103-114) ---------------------------------------
class UVLayout:
    """The UV layout of the textured flows: ``BFM_UV.npy`` (nver, >=2) UV coordinates, ``keptInd.npy`` the kept vertices
    and ``deletedTri.npy`` the (3, ntri) 1-based triangles over them.  The texel coordinates are numpy's, in the array's
    own dtype, as the scripts compute them: ``coord_u = (uv[:,1]*255.0).astype(np.int32)`` (row) and ``coord_v =
    (uv[:,0]*255.0).astype(np.int32)`` (column).  Every refusal happens here or in :meth:`texels`, before any CUDA call."""

    def __init__(self, bfm_uv, keep, deleted_tri):
        uv = np.asarray(bfm_uv)
        if uv.ndim != 2 or uv.shape[1] < 2 or uv.shape[0] < 1 or uv.dtype.kind != 'f':
            raise ValueError(f'BFM_UV must be a float (nver, 2) array, got {uv.dtype} {uv.shape}')
        with np.errstate(invalid='ignore', over='ignore'):
            self.coord_u = (uv[:, 1] * 255.0).astype(np.int32)
            self.coord_v = (uv[:, 0] * 255.0).astype(np.int32)
        self.nver = int(uv.shape[0])
        k = np.asarray(keep)
        if k.ndim != 1 or k.dtype.kind not in 'iu' or k.size < 1:
            raise ValueError(f'keptInd must be a non-empty 1-d integer array, got {k.dtype} {k.shape}')
        bad = np.argwhere((k < 0) | (k >= self.nver))
        if bad.size:
            raise ValueError(f'keptInd[{int(bad[0, 0])}] = {int(k[bad[0, 0]])} lies outside [0, {self.nver})')
        self.keep = np.ascontiguousarray(k, dtype=np.int64)
        self.n_keep = int(k.size)
        tri = np.asarray(deleted_tri)
        if tri.ndim != 2 or tri.shape[0] != 3 or tri.shape[1] < 1 or tri.dtype.kind not in 'iu':
            raise ValueError(f'deletedTri must be a (3, ntri) integer array, got {tri.dtype} {tri.shape}')
        bad = np.argwhere((tri < 1) | (tri > self.n_keep))
        if bad.size:
            i, j = (int(x) for x in bad[0])
            raise ValueError(f'deletedTri[{i}, {j}] - 1 = {int(tri[i, j]) - 1} lies outside [0, {self.n_keep}) kept vertices')
        self.deleted_tri = tri                                               # written as given by write_obj_with_colors
        self.render_tri = np.ascontiguousarray((tri.astype(np.int64) - 1).T, dtype=np.int32)   # connectivity=deletedTri-1, (ntri,3)
        self._texels = {}

    @classmethod
    def load(cls, directory: str) -> 'UVLayout':
        """The layout of a ``3dmm_data`` directory: ``BFM_UV.npy``, ``keptInd.npy``, ``deletedTri.npy``."""
        import os
        return cls(*(np.load(os.path.join(directory, f)) for f in ('BFM_UV.npy', 'keptInd.npy', 'deletedTri.npy')))

    def texels(self, h: int, w: int, what: str = 'the UV map') -> np.ndarray:
        """(n_keep, 2) int32 (row, column) of the unflipped (h, w) map that ``np.flip(map, 0)[coord_u, coord_v][keep]``
        reads: row r in [-h, h) is row ``h-1-(r mod h)``, column c in [-w, w) is column ``c mod w``.  As the reference
        indexes every vertex before it applies ``keep``, a coordinate outside those ranges raises ``IndexError`` for any
        vertex, kept or not, naming it and ``what``."""
        key = (int(h), int(w))
        if key not in self._texels:
            h, w = key
            for axis, c, n in ((0, self.coord_u, h), (1, self.coord_v, w)):
                bad = np.argwhere((c < -n) | (c >= n))
                if bad.size:
                    i = int(bad[0, 0])
                    raise IndexError(f'vertex {i}: index {int(c[i])} is out of bounds for axis {axis} with size {n} of {what} '
                                     f'({h}x{w})')
            rows = h - 1 - np.mod(self.coord_u[self.keep].astype(np.int64), h)
            cols = np.mod(self.coord_v[self.keep].astype(np.int64), w)
            self._texels[key] = np.ascontiguousarray(np.stack([rows, cols], 1), dtype=np.int32)
        return self._texels[key]


def uv_maps_host(maps, n_images: int, overlay: bool) -> list:
    """The UV maps of a call as a list of (h, w, 3) uint8 host arrays, one per image (``maps``: one (h, w, 3|4) map per
    image, or one map for all of them).  A 4-channel map keeps channels 0..2, all that ``write_obj_with_colors`` prints;
    the overlay refuses it, as the reference's ``texture *= light`` cannot broadcast it.  Grayscale and non-uint8 maps
    raise ValueError."""
    def host(m):
        m = m.cpu().numpy() if hasattr(m, 'cpu') else np.asarray(m)
        if m.dtype != np.uint8:
            raise ValueError(f'UV maps must be uint8 (what cv2.imread(path, -1) gives for an 8-bit PNG), got {m.dtype}')
        if m.ndim != 3 or m.shape[2] not in (3, 4) or m.shape[0] < 1 or m.shape[1] < 1:
            raise ValueError(f'UV maps must be (h, w, 3) or (h, w, 4) colour images, got {m.shape}')
        if m.shape[2] == 4:
            if overlay:
                raise ValueError('a 4-channel UV map cannot texture the overlay: the reference\'s `texture *= light` does not '
                                 'broadcast (n, 4) against (n, 3)')
            m = m[:, :, :3]
        return np.ascontiguousarray(m)
    one = (hasattr(maps, 'ndim') and maps.ndim == 3) or (hasattr(maps, 'shape') and len(maps.shape) == 3)
    maps = [host(maps)] if one else [host(m) for m in maps]
    if len(maps) != n_images and len(maps) != 1:
        raise ValueError(f'{len(maps)} UV maps for {n_images} images: give one map per image, or one for all of them')
    return maps


class UVMaps:
    """UV maps on one device and the texels of a :class:`UVLayout` resolved for each of their sizes, uploaded in one copy:
    :meth:`sample` gives the textures and colours of ``syn_uv_sample`` for faces a..b-1, face f reading map
    ``face_map[f]``."""

    def __init__(self, layout: UVLayout, maps, face_map, device):
        import torch
        self.layout, self.device = layout, torch.device(device)
        self.face_map = np.ascontiguousarray(face_map, dtype=np.int32).reshape(-1)
        n = len(maps)
        if self.face_map.size and (self.face_map.min() < 0 or self.face_map.max() >= n):
            raise ValueError(f'face_map names maps outside [0, {n})')
        self.texels = np.ascontiguousarray(np.stack([layout.texels(m.shape[0], m.shape[1], f'UV map {i}') for i, m in enumerate(maps)]))
        sizes = [3 * m.shape[0] * m.shape[1] for m in maps]
        offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        self.table = np.array([[offs[i], m.shape[0], m.shape[1]] for i, m in enumerate(maps)], np.int64).reshape(n, 3)
        self.n_maps, self.map_bytes = n, int(offs[-1])
        # one int64 buffer: table (n,3) | texels (n, n_keep, 2) int32 | face_map int32 | the map bytes
        a = 3 * n
        b = a + self.texels.size // 2
        c = b + (self.face_map.size + 1) // 2
        buf = np.zeros(c + (self.map_bytes + 7) // 8, np.int64)
        buf[:a] = self.table.reshape(-1)
        buf[a:b].view(np.int32)[:] = self.texels.reshape(-1)
        buf[b:c].view(np.int32)[:self.face_map.size] = self.face_map
        buf[c:].view(np.uint8)[:self.map_bytes] = np.concatenate([m.reshape(-1) for m in maps])
        self.dev = torch.from_numpy(buf).to(self.device)
        self._parts = (a, b, c)
        self.launches = 0

    def sample(self, a: int, b: int, texture: bool = True, colors: bool = False):
        """``(texture, colors)`` of faces a..b-1: float32 (b-a, n_keep, 3) ``colors_uv[keep] / 255`` and int64 (b-a, n_keep,
        3) ``colors_uv[keep]``, each None unless asked for."""
        import torch
        from . import _lib
        pa, pb, pc = self._parts
        k = self.layout.n_keep
        tex = torch.empty((b - a, k, 3), dtype=torch.float32, device=self.device) if texture else None
        col = torch.empty((b - a, k, 3), dtype=torch.int64, device=self.device) if colors else None
        fm = np.ascontiguousarray(self.face_map[a:b])
        fm_dev = self.dev[pb:].view(torch.int32)[a:b]
        _lib.launch(self.device, 'syn_uv_sample', self.dev[pc:].data_ptr(), self.map_bytes, self.table.ctypes.data,
                    self.dev.data_ptr(), self.n_maps, self.texels.ctypes.data, self.dev[pa:].data_ptr(), k, fm.ctypes.data,
                    fm_dev.data_ptr(), b - a, None if tex is None else tex.data_ptr(), None if col is None else col.data_ptr())
        self.launches += 1
        return tex, col
