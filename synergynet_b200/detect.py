"""FaceBoxes post-processing on the H100 (SURVEY.md section 8 row f3): prior boxes, box decode, score filter, ordering
and greedy NMS in ``libsynergy_b200.so`` (``csrc/kernels_detect.cuh``, NMS kernels in ``csrc/kernels_render.cuh``).

Reference-shaped surface: :func:`nms` has the signature and return value of ``FaceBoxes/utils/nms_wrapper.py:13-18``
(whose Cython backend does not build with current Cython / numpy, SURVEY.md section 8(c)); :func:`cpu_nms` /
:func:`py_cpu_nms` are the two comparison conventions the reference ships; :func:`detect_postprocess` is
``FaceBoxes.__call__`` from the network outputs on (``FaceBoxes/FaceBoxes.py:98-143``).  The detector CNN itself is not
part of this library.  No CPU fallback.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

# FaceBoxes/FaceBoxes.py:17-22
confidence_threshold = 0.05
top_k = 5000
keep_top_k = 750
nms_threshold = 0.3
vis_thres = 0.5


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError('synergynet_b200.detect needs a CUDA device (H100, sm_90a); there is no CPU fallback')
    return torch.device('cuda', torch.cuda.current_device())


def nms_device(dets: torch.Tensor, thresh: float, mode: int = _lib.NMS_CPU_NMS, n: int = None):
    """Greedy NMS of ``dets`` (N,5) float32 CUDA rows ``[x1 y1 x2 y2 score]`` already in descending score order (only the
    first ``n`` rows if given).  Returns ``(keep, n_keep)`` device tensors: kept row indices in order, and their count."""
    if dets.dtype != torch.float32 or dets.dim() != 2 or dets.shape[1] != 5 or not dets.is_cuda or not dets.is_contiguous():
        raise ValueError('dets must be a contiguous float32 (N,5) CUDA tensor')
    n = int(dets.shape[0]) if n is None else int(n)
    words = (n + 63) // 64
    mask = torch.empty((max(n * words, 1),), dtype=torch.int64, device=dets.device)
    keep = torch.empty((max(n, 1),), dtype=torch.int32, device=dets.device)
    n_keep = torch.zeros((1,), dtype=torch.int32, device=dets.device)
    _lib.launch(dets.device, 'syn_nms', dets.data_ptr(), n, float(thresh), int(mode), mask.data_ptr(), keep.data_ptr(),
                n_keep.data_ptr())
    return keep, n_keep


def _nms_numpy(dets: np.ndarray, thresh: float, mode: int):
    if dets.shape[0] == 0:
        return []
    d = np.ascontiguousarray(dets, dtype=np.float32)
    order = d[:, 4].argsort()[::-1]                         # both reference functions re-sort by score first
    dev = torch.from_numpy(np.ascontiguousarray(d[order])).to(_device())
    keep, n_keep = nms_device(dev, thresh, mode)
    k = keep[:int(n_keep.item())].cpu().numpy()
    return [int(i) for i in order[k]]


def cpu_nms(dets: np.ndarray, thresh: float):
    """``FaceBoxes/utils/nms/cpu_nms.pyx:17-68``: indices of the kept rows of ``dets`` (N,5), suppression on ``ovr >= thresh``."""
    return _nms_numpy(dets, thresh, _lib.NMS_CPU_NMS)


def py_cpu_nms(dets: np.ndarray, thresh: float):
    """``FaceBoxes/utils/nms/py_cpu_nms.py:10-38``: the same with ``ovr <= thresh`` kept (float32 comparison)."""
    return _nms_numpy(dets, thresh, _lib.NMS_PY_CPU_NMS)


def nms(dets, thresh):
    """``FaceBoxes/utils/nms_wrapper.py:13-18``."""
    if dets.shape[0] == 0:
        return []
    return cpu_nms(dets, thresh)


def num_priors(im_height: int, im_width: int) -> int:
    return int(_lib.load().syn_faceboxes_num_priors(int(im_height), int(im_width)))


def decode_device(loc: torch.Tensor, conf: torch.Tensor, im_height: int, im_width: int, scale: float = 1.0,
                  conf_thresh: float = confidence_threshold, k: int = top_k):
    """``FaceBoxes.py:98-121`` on the device: ``loc`` (P,4), ``conf`` (P,2) float32 CUDA tensors (network outputs for an
    ``im_height`` x ``im_width`` input) -> ``(dets, n)``: (k,5) rows ``[x1 y1 x2 y2 score]`` in descending score order in
    original-image pixels, of which the first ``n`` (device int32) are valid."""
    p = num_priors(im_height, im_width)
    loc, conf = loc.reshape(-1, 4).contiguous(), conf.reshape(-1, 2).contiguous()
    if loc.shape[0] != p or conf.shape[0] != p or loc.dtype != torch.float32 or conf.dtype != torch.float32 or not loc.is_cuda:
        raise ValueError(f'loc / conf must be float32 CUDA tensors with {p} priors for a {im_height}x{im_width} input')
    cand = torch.empty((p + 1,), dtype=torch.int32, device=loc.device)
    dets = torch.zeros((k, 5), dtype=torch.float32, device=loc.device)
    n = torch.zeros((1,), dtype=torch.int32, device=loc.device)
    _lib.launch(loc.device, 'syn_faceboxes_decode', loc.data_ptr(), conf.data_ptr(), int(im_height), int(im_width), float(im_width),
                float(im_height), float(scale), float(conf_thresh), int(k), cand.data_ptr(), dets.data_ptr(), n.data_ptr())
    return dets, n


def decode_batch_device(loc: torch.Tensor, conf: torch.Tensor, im_height: int, im_width: int, scale: float = 1.0,
                        conf_thresh: float = confidence_threshold, k: int = top_k):
    """:func:`decode_device` for N frames of one size in the same two launches: ``loc`` (N,P,4), ``conf`` (N,P,2) ->
    ``(dets, n)``: (N,k',5) and (N,) device int32, frame i's block and count being what ``decode_device`` gives for
    ``loc[i]``, ``conf[i]``.  k' = min(k, P): a frame cannot have more candidates than priors."""
    p = num_priors(im_height, im_width)
    if loc.dim() != 3 or conf.dim() != 3 or tuple(loc.shape[1:]) != (p, 4) or tuple(conf.shape) != (loc.shape[0], p, 2) or \
            loc.shape[0] == 0 or loc.dtype != torch.float32 or conf.dtype != torch.float32 or not loc.is_cuda or conf.device != loc.device:
        raise ValueError(f'loc / conf must be float32 CUDA tensors (N,{p},4) / (N,{p},2) for {im_height}x{im_width} inputs')
    loc, conf = loc.contiguous(), conf.contiguous()
    nf, k = int(loc.shape[0]), min(int(k), p)
    cand = torch.empty((nf, p + 1), dtype=torch.int32, device=loc.device)
    dets = torch.zeros((nf, k, 5), dtype=torch.float32, device=loc.device)
    n = torch.zeros((nf,), dtype=torch.int32, device=loc.device)
    _lib.launch(loc.device, 'syn_faceboxes_decode_batch', loc.data_ptr(), conf.data_ptr(), nf, int(im_height), int(im_width),
                float(im_width), float(im_height), float(scale), float(conf_thresh), k, cand.data_ptr(), dets.data_ptr(), n.data_ptr())
    return dets, n


def decode_images_device(loc: torch.Tensor, conf: torch.Tensor, sizes, scales, conf_thresh: float = confidence_threshold,
                         k: int = top_k):
    """:func:`decode_device` for N network inputs of any sizes in the same two launches: ``loc`` (sum P_i,4), ``conf``
    (sum P_i,2) as ``FaceBoxesNet`` packs them, ``sizes`` the N (h, w) inputs, ``scales`` their shrink factors ->
    ``(dets, n)``: (N,k',5) and (N,) device int32, image i's block and count being what ``decode_device`` gives for its
    priors alone.  k' = min(k, max P_i)."""
    hw = np.ascontiguousarray(np.array(sizes, np.int32).reshape(-1, 2))
    hs, ws = np.ascontiguousarray(hw[:, 0]), np.ascontiguousarray(hw[:, 1])
    sc = np.ascontiguousarray(scales, dtype=np.float32).reshape(-1)
    nf = int(hw.shape[0])
    if nf == 0 or sc.shape[0] != nf or (hw < 1).any():
        raise ValueError(f'{nf} image sizes (each >= 1) and {sc.shape[0]} scales: one of each per image, at least one image')
    ps = [num_priors(h, w) for h, w in hw.tolist()]
    if loc.dim() != 2 or conf.dim() != 2 or tuple(loc.shape) != (sum(ps), 4) or tuple(conf.shape) != (sum(ps), 2) or \
            loc.dtype != torch.float32 or conf.dtype != torch.float32 or not loc.is_cuda or conf.device != loc.device:
        raise ValueError(f'loc / conf must be float32 CUDA tensors ({sum(ps)},4) / ({sum(ps)},2) for these {nf} inputs')
    loc, conf = loc.contiguous(), conf.contiguous()
    k = min(int(k), max(ps))
    cand = torch.empty((nf + sum(ps),), dtype=torch.int32, device=loc.device)
    dets = torch.zeros((nf, k, 5), dtype=torch.float32, device=loc.device)
    n = torch.zeros((nf,), dtype=torch.int32, device=loc.device)
    _lib.launch(loc.device, 'syn_faceboxes_decode_images', loc.data_ptr(), conf.data_ptr(), nf, hs.ctypes.data, ws.ctypes.data,
                sc.ctypes.data, float(conf_thresh), k, cand.data_ptr(), dets.data_ptr(), n.data_ptr())
    return dets, n


def nms_batch_device(dets: torch.Tensor, n: torch.Tensor, thresh: float, mode: int = _lib.NMS_CPU_NMS):
    """:func:`nms_device` per frame without a host round trip: ``dets`` (N,K,5) in descending score order per frame, ``n``
    (N,) device int32 counts (``decode_batch_device``'s outputs).  Returns ``(keep (N,K) int32, n_keep (N,) int32)``; the
    first ``n_keep[i]`` entries of ``keep[i]`` are frame i's kept rows, the rest is not written."""
    if dets.dtype != torch.float32 or dets.dim() != 3 or dets.shape[2] != 5 or dets.shape[0] == 0 or dets.shape[1] == 0 or \
            not dets.is_cuda or not dets.is_contiguous():
        raise ValueError('dets must be a contiguous float32 (N,K,5) CUDA tensor')
    nf, rows = int(dets.shape[0]), int(dets.shape[1])
    if n.dtype != torch.int32 or tuple(n.shape) != (nf,) or n.device != dets.device or not n.is_contiguous():
        raise ValueError(f'n must be the ({nf},) int32 counts on the device of dets')
    mask = torch.empty((nf * rows * ((rows + 63) // 64),), dtype=torch.int64, device=dets.device)
    keep = torch.empty((nf, rows), dtype=torch.int32, device=dets.device)
    n_keep = torch.zeros((nf,), dtype=torch.int32, device=dets.device)
    _lib.launch(dets.device, 'syn_nms_batch', dets.data_ptr(), n.data_ptr(), nf, rows, float(thresh), int(mode), mask.data_ptr(),
                keep.data_ptr(), n_keep.data_ptr())
    return keep, n_keep


def detect_postprocess(loc, conf, im_height: int, im_width: int, scale: float = 1.0):
    """``FaceBoxes.__call__`` after the forward pass (``FaceBoxes/FaceBoxes.py:98-143``): list of
    ``[xmin, ymin, xmax, ymax, score]`` with score above ``vis_thres``, at most ``keep_top_k`` after NMS."""
    dev = _device()
    loc = torch.as_tensor(loc, dtype=torch.float32).to(dev)
    conf = torch.as_tensor(conf, dtype=torch.float32).to(dev)
    dets, n = decode_device(loc, conf, im_height, im_width, scale)
    n_host = int(n.item())
    if n_host == 0:
        return []
    keep, n_keep = nms_device(dets, nms_threshold, _lib.NMS_CPU_NMS, n=n_host)
    kept = dets[keep[:int(n_keep.item())].long()][:keep_top_k].cpu().numpy()
    return [[b[0], b[1], b[2], b[3], b[4]] for b in kept if b[4] > vis_thres]
