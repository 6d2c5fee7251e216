"""Host-side API semantics around the hot path, batched (reference ``utils/inference.py``).

Only tiny per-face affine / pose algebra, the integer ROI crop (the host restatement the tests compare against) and its
device twin ``crop_resize_device`` live here; vertex reconstruction itself runs on the GPU (``Engine.reconstruct``).
"""
from __future__ import annotations

from typing import Sequence, Tuple

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
    with torch.cuda.device(image.device):
        _lib.check(_lib.load().syn_crop_resize(image.data_ptr(), image.shape[0], image.shape[1], image.shape[2], plan.data_ptr(), B,
                                               out_h, out_w, interpolation, out.data_ptr(), *strides,
                                               torch.cuda.current_stream(image.device).cuda_stream))
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
    with torch.cuda.device(frames.device):
        _lib.check(_lib.load().syn_crop_resize_batch(frames.data_ptr(), frames.shape[0], frames.shape[1], frames.shape[2],
                                                     frames.shape[3], plan.data_ptr(), B, out_h, out_w, interpolation,
                                                     out.data_ptr(), *strides, torch.cuda.current_stream(frames.device).cuda_stream))
    return out


def stack_frames_host(frames) -> np.ndarray:
    """N equally sized (H,W,3) BGR images (a list, or one (N,H,W,3) array) -> one contiguous uint8 (N,H,W,3) array."""
    if not (isinstance(frames, np.ndarray) and frames.ndim == 4):
        frames = [np.asarray(f) for f in frames]
        if not frames:
            raise ValueError('no frames: a frame batch needs at least one image')
        shapes = [tuple(f.shape) for f in frames]
        if any(sh != shapes[0] for sh in shapes):
            sizes = ', '.join('x'.join(str(d) for d in sh) for sh in sorted(set(shapes)))
            raise ValueError(f'the frames of one batch must have one size, got {sizes}; group the frames by size')
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


def decompose_camera(P: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Batched P2sRt (utils/inference.py:33-43): P (B,3,4) -> scale (B,), R (B,3,3), t (B,3)."""
    r1, r2 = P[:, 0, :3], P[:, 1, :3]
    n1 = np.linalg.norm(r1, axis=1, keepdims=True)
    n2 = np.linalg.norm(r2, axis=1, keepdims=True)
    u1, u2 = r1 / n1, r2 / n2
    R = np.stack([u1, u2, np.cross(u1, u2)], axis=1)
    return ((n1 + n2) / 2.0)[:, 0], R, P[:, :, 3]


def rotation_to_euler_deg(R: np.ndarray) -> np.ndarray:
    """Batched matrix2angle_corr (utils/inference.py:45-62) -> (B,3) degrees."""
    r20 = R[:, 2, 0]
    lock = (r20 == 1) | (r20 == -1)
    x = np.arcsin(np.clip(r20, -1, 1))
    cx = np.where(lock, 1.0, np.cos(x))
    y = np.arctan2(R[:, 1, 2] / cx, R[:, 2, 2] / cx)
    z = np.arctan2(R[:, 0, 1] / cx, R[:, 0, 0] / cx)
    neg = r20 == -1
    x = np.where(lock, np.where(neg, np.pi / 2, -np.pi / 2), x)
    y = np.where(lock, np.where(neg, np.arctan2(R[:, 0, 1], R[:, 0, 2]),
                                np.arctan2(-R[:, 0, 1], -R[:, 0, 2])), y)
    z = np.where(lock, 0.0, z)
    return np.stack([x, y, z], 1) * (180.0 / np.pi)


def predict_pose_batch(params: np.ndarray, param_mean: np.ndarray, param_std: np.ndarray,
                       roi_boxes: Sequence[Sequence[float]]):
    """parse_pose + predict_pose (utils/inference.py:86-92,146-157) for B whitened vectors.
    Returns a list of ``[angles(list of 3), t3d(ndarray 3)]`` like the reference."""
    p = params * param_std[:62] + param_mean[:62]
    cam = p[:, :12].reshape(-1, 3, 4)
    _, R, t3d = decompose_camera(cam)
    ang = rotation_to_euler_deg(R)
    out = []
    for i, box in enumerate(roi_boxes):
        sx, sy, ex, ey = box[:4]
        t = t3d[i].copy()
        t[0] = t[0] * ((ex - sx) / STD_SIZE) + sx
        t[1] = t[1] * ((ey - sy) / STD_SIZE) + sy
        out.append([[float(a) for a in ang[i]], t])
    return out


# lighting of the solid-mesh overlay (utils/render.py:18-27), consumed by synergynet_b200.Sim3DR.render
RENDER_CFG = {
    'intensity_ambient': 0.75, 'color_ambient': (1, 1, 1),
    'intensity_directional': 0.7, 'color_directional': (1, 1, 1),
    'intensity_specular': 0.2, 'specular_exp': 5,
    'light_pos': (0, 0, 5), 'view_pos': (0, 0, 5),
}
