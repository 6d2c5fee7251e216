"""The FaceBoxes detector on the H100 (SURVEY.md section 8 row f3): network, box decode and NMS all on the device.

Reference-shaped surface: :class:`FaceBoxes` has the constructor and call signature of ``FaceBoxes/FaceBoxes.py:46-143``
(``FaceBoxes(timer_flag=False)``, ``face_boxes(img_bgr_uint8) -> [[xmin, ymin, xmax, ymax, score], ...]``) and loads the
reference's checkpoint schema (``FaceBoxes/models/faceboxes.py``: ``conv1.conv.weight``, ``inception2.branch3x3.bn.*``,
``loc.0.bias`` ..., optional ``module.`` prefix, ``utils/functions.py:19-43``).  The 33 convolutions, the pools and the
softmax run in ``libsynergy_b200.so`` (``csrc/kernels_detect.cuh``); :meth:`FaceBoxes.detect_batch` runs them on a stack of
equally sized frames in the same launches, with one host synchronisation for the whole stack.  An image above 720 x 1080 is uploaded as it is
and shrunk on the device (``inference.crop_resize_device``, ``csrc/kernels_resize.cuh``) to the bytes the reference's
``cv2.resize`` makes on the host.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib, detect
from .engine import Handle
from .inference import (INTER_LINEAR, ImagePack, chunk_ranges, crop_resize_device, crop_resize_frames_device, crop_resize_images_device,
                        pack_images, stack_frames_device)

# FaceBoxes/FaceBoxes.py:24-25
scale_flag = True
HEIGHT, WIDTH = 720, 1080


def shrink_size(h: int, w: int):
    """``(scale, (out_w, out_h))`` of the detector's shrink of an h x w image (FaceBoxes/FaceBoxes.py:62-79): the
    image's own size at scale 1 when it fits in HEIGHT x WIDTH (or ``scale_flag`` is off), else cv2.resize's dsize."""
    scale = 1
    if scale_flag:
        if h > HEIGHT:
            scale = HEIGHT / h
        if w * scale > WIDTH:
            scale *= WIDTH / (w * scale)
    return scale, ((int(scale * w), int(scale * h)) if scale != 1 else (w, h))


def layer_plan() -> List[dict]:
    """The 33 convolutions in execution order as the library reports them (name = state_dict prefix)."""
    lib = _lib.load()
    out = []
    for i in range(lib.syn_fb_num_layers()):
        d = _lib.FbLayerDesc()
        _lib.check(lib.syn_fb_layer_desc(i, C.byref(d)))
        out.append(dict(index=i, name=d.name.decode(), cin=d.cin, cout=d.cout, ksize=d.ksize, stride=d.stride, pad=d.pad,
                        has_bn=bool(d.has_bn), activation=d.activation))
    return out


def state_dict_keys() -> List[str]:
    """Keys of a ``FaceBoxesNet`` state dict (faceboxes.py:8-18, 50-58, 94-106)."""
    keys = []
    for L in layer_plan():
        if L['has_bn']:
            keys.append(f"{L['name']}.conv.weight")
            keys += [f"{L['name']}.bn.{k}" for k in ('weight', 'bias', 'running_mean', 'running_var', 'num_batches_tracked')]
        else:
            keys += [f"{L['name']}.weight", f"{L['name']}.bias"]
    return keys


class FaceBoxesNet(Handle):
    """Device-side detector network: one ``syn_fb_t`` handle."""
    _CREATE, _DESTROY = 'syn_fb_create', 'syn_fb_destroy'

    def __init__(self, state_dict: Dict[str, torch.Tensor], device=None):
        self._lib = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError('synergynet_b200.faceboxes needs a CUDA device (H100, sm_90a); there is no CPU fallback')
        super().__init__(torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device))
        sd = {(k[7:] if k.startswith('module.') else k): v for k, v in state_dict.items()}       # utils/functions.py:19-24
        f32 = lambda t: torch.as_tensor(t).detach().to(device='cpu', dtype=torch.float32).contiguous()
        for L in layer_plan():
            n = L['name']
            if L['has_bn']:
                w = f32(sd[f'{n}.conv.weight'])
                bn = [f32(sd[f'{n}.bn.{k}']) for k in ('weight', 'bias', 'running_mean', 'running_var')]
                _lib.check(self._lib.syn_fb_set_layer(self._h, L['index'], w.data_ptr(), w.numel(), None,
                                                      *[t.data_ptr() for t in bn], 1e-5))
            else:
                w, b = f32(sd[f'{n}.weight']), f32(sd[f'{n}.bias'])
                _lib.check(self._lib.syn_fb_set_layer(self._h, L['index'], w.data_ptr(), w.numel(), b.data_ptr(), None, None, None, None, 0.0))
        _lib.check(self._lib.syn_fb_commit(self._h))

    @property
    def launch_count(self) -> int:
        return int(self._lib.syn_fb_launch_count(self._h))

    def forward(self, image: torch.Tensor):
        """``image`` (H,W,3) uint8 BGR on the device -> ``(loc (P,4), conf (P,2))`` like ``FaceBoxesNet.forward`` in 'test'
        phase (faceboxes.py:112-150) applied to ``img - (104,117,123)``."""
        if image.dtype != torch.uint8 or image.dim() != 3 or image.shape[2] != 3 or image.device != self.device or not image.is_contiguous():
            raise ValueError('image must be a contiguous uint8 (H,W,3) tensor on the detector device')
        h, w = int(image.shape[0]), int(image.shape[1])
        p = detect.num_priors(h, w)
        loc = torch.empty((p, 4), dtype=torch.float32, device=self.device)
        conf = torch.empty((p, 2), dtype=torch.float32, device=self.device)
        self._call('syn_fb_forward', image.data_ptr(), h, w, loc.data_ptr(), conf.data_ptr())
        return loc, conf

    def debug_fill_workspaces(self, byte: int) -> int:
        """Set every byte of the detector's activation workspace, at its allocated size, to ``byte`` and clear its
        geometry table, ordered on the current stream after the previous call; returns the number of bytes written.
        Poisoned-workspace tests only."""
        n = C.c_size_t(0)
        self._call('syn_fb_debug_fill_workspaces', int(byte), C.byref(n))
        return int(n.value)

    def debug_fill_on_grow(self, byte: int) -> None:
        """Every later workspace growth sets its new buffers to ``byte`` (-1: off).  Poisoned-workspace tests only."""
        self._call_host('syn_fb_debug_fill_on_grow', int(byte))

    def debug_forward_until(self, image: torch.Tensor, stage: int) -> torch.Tensor:
        """Run :meth:`forward`'s launch sequence up to launch ``stage`` (0..38, table at ``syn_fb_debug_forward_until`` in
        include/synergy_b200.h) and return the whole tensor that launch wrote: an NHWC ``(h, w, channels)`` map, or the
        flat ``loc`` (P*4) / ``conf`` (P*2) for stages 32..38.  ``loc`` / ``conf`` start as NaN, so what a head did not
        write reads NaN.  Per-stage tests only."""
        if image.dtype != torch.uint8 or image.dim() != 3 or image.shape[2] != 3 or image.device != self.device or not image.is_contiguous():
            raise ValueError('image must be a contiguous uint8 (H,W,3) tensor on the detector device')
        h, w = int(image.shape[0]), int(image.shape[1])
        p = detect.num_priors(h, w)
        loc = torch.full((p * 4,), float('nan'), dtype=torch.float32, device=self.device)
        conf = torch.full((p * 2,), float('nan'), dtype=torch.float32, device=self.device)
        shape = debug_stage_shape(stage, h, w)
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        self._call('syn_fb_debug_forward_until', image.data_ptr(), h, w, stage, out.data_ptr(), out.numel(), loc.data_ptr(),
                   conf.data_ptr())
        return out

    def _check_stack(self, images: torch.Tensor):
        if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] != 3 or \
                images.shape[0] == 0 or images.device != self.device or not images.is_contiguous():
            raise ValueError('images must be a contiguous uint8 (N,H,W,3) tensor with N >= 1 on the detector device')
        if images.shape[0] > _lib.FB_MAX_FRAMES:
            raise ValueError(f'{images.shape[0]} frames in one call, at most {_lib.FB_MAX_FRAMES} (FaceBoxes.detect_batch splits a stack)')
        return int(images.shape[0]), int(images.shape[1]), int(images.shape[2])

    def forward_batch(self, images: torch.Tensor):
        """:meth:`forward` for a stack of frames in the same 39 launches: ``images`` (N,H,W,3) uint8 BGR on the device ->
        ``(loc (N,P,4), conf (N,P,2))``; ``loc[i]``, ``conf[i]`` have the bits of ``forward(images[i])``."""
        n, h, w = self._check_stack(images)
        p = detect.num_priors(h, w)
        loc = torch.empty((n, p, 4), dtype=torch.float32, device=self.device)
        conf = torch.empty((n, p, 2), dtype=torch.float32, device=self.device)
        self._call('syn_fb_forward_batch', images.data_ptr(), n, h, w, loc.data_ptr(), conf.data_ptr())
        return loc, conf

    def debug_forward_batch_until(self, images: torch.Tensor, stage: int) -> torch.Tensor:
        """:meth:`debug_forward_until` on :meth:`forward_batch`'s launch sequence: the ``(N, h, w, channels)`` stack of the
        maps launch ``stage`` wrote, or the ``(N, P*4)`` loc / ``(N, P*2)`` conf for stages 32..38 (NaN where no head has
        written yet).  Per-stage tests only."""
        n, h, w = self._check_stack(images)
        p = detect.num_priors(h, w)
        loc = torch.full((n, p * 4), float('nan'), dtype=torch.float32, device=self.device)
        conf = torch.full((n, p * 2), float('nan'), dtype=torch.float32, device=self.device)
        out = torch.empty((n,) + tuple(debug_stage_shape(stage, h, w)), dtype=torch.float32, device=self.device)
        self._call('syn_fb_debug_forward_batch_until', images.data_ptr(), n, h, w, stage, out.data_ptr(), out.numel(),
                   loc.data_ptr(), conf.data_ptr())
        return out

    def _check_images(self, images):
        """A list of contiguous (h,w,3) uint8 CUDA tensors on the detector device, or an ImagePack there -> ImagePack."""
        if isinstance(images, ImagePack):
            if images.data.device != self.device or images.data.dtype != torch.uint8 or not images.data.is_contiguous():
                raise ValueError(f'packed images must be contiguous uint8 on the detector device {self.device}, got '
                                 f'{images.data.dtype} on {images.data.device}')
        else:
            images = list(images)
            for im in images:
                if not isinstance(im, torch.Tensor) or im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3 or \
                        im.device != self.device or not im.is_contiguous():
                    raise ValueError('images must be contiguous uint8 (H,W,3) tensors on the detector device')
            images = pack_images(images, self.device)
        if not 1 <= len(images) <= _lib.FB_MAX_FRAMES:
            raise ValueError(f'{len(images)} images in one call, 1..{_lib.FB_MAX_FRAMES} (FaceBoxes.detect_images splits a list)')
        return images

    def forward_packed(self, images):
        """:meth:`forward` for N images of any sizes in the same 39 launches: ``images`` a list of (h_i,w_i,3) uint8 CUDA
        tensors or an :class:`ImagePack` -> ``(loc (sum P_i,4), conf (sum P_i,2), p)``, image i's priors being rows
        ``p[i]:p[i+1]``."""
        pack = self._check_images(images)
        p = np.concatenate([[0], np.cumsum([detect.num_priors(h, w) for h, w in pack.sizes])]).astype(int).tolist()
        loc = torch.empty((p[-1], 4), dtype=torch.float32, device=self.device)
        conf = torch.empty((p[-1], 2), dtype=torch.float32, device=self.device)
        hs, ws = pack.arrays()
        self._call('syn_fb_forward_images', pack.data.data_ptr(), len(pack), hs.ctypes.data, ws.ctypes.data, loc.data_ptr(),
                   conf.data_ptr())
        return loc, conf, p

    def forward_images(self, images):
        """:meth:`forward` for N images of any sizes in the same 39 launches: a list of contiguous (h_i,w_i,3) uint8 CUDA
        tensors -> lists of ``(P_i,4)`` loc and ``(P_i,2)`` conf views, entry i having the bits of ``forward(images[i])``."""
        loc, conf, p = self.forward_packed(images)
        return [loc[a:b] for a, b in zip(p[:-1], p[1:])], [conf[a:b] for a, b in zip(p[:-1], p[1:])]

    def debug_forward_images_until(self, images, stage: int) -> list:
        """:meth:`debug_forward_until` on :meth:`forward_images`'s launch sequence: one tensor per image, shaped as
        ``debug_forward_until`` returns it for that image alone.  Per-stage tests only."""
        pack = self._check_images(images)
        shapes = [debug_stage_shape(stage, h, w) for h, w in pack.sizes]
        p = sum(detect.num_priors(h, w) for h, w in pack.sizes)
        loc = torch.full((p * 4,), float('nan'), dtype=torch.float32, device=self.device)
        conf = torch.full((p * 2,), float('nan'), dtype=torch.float32, device=self.device)
        numel = [int(np.prod(sh)) for sh in shapes]
        out = torch.empty((sum(numel),), dtype=torch.float32, device=self.device)
        hs, ws = pack.arrays()
        self._call('syn_fb_debug_forward_images_until', pack.data.data_ptr(), len(pack), hs.ctypes.data, ws.ctypes.data, stage,
                   out.data_ptr(), out.numel(), loc.data_ptr(), conf.data_ptr())
        at = np.concatenate([[0], np.cumsum(numel)]).astype(int).tolist()
        return [out[a:b].view(sh) for a, b, sh in zip(at[:-1], at[1:], shapes)]


def _conv_out(n: int, k: int, s: int, p: int) -> int:
    return (n + 2 * p - k) // s + 1


def debug_stage_shape(stage: int, h: int, w: int) -> tuple:
    """Shape of the tensor launch ``stage`` of the detector writes, for an h x w image (see ``debug_forward_until``)."""
    if not 0 <= stage < 39:
        raise ValueError(f'detector stage {stage} outside 0..38')
    h1, w1 = _conv_out(h, 7, 4, 3), _conv_out(w, 7, 4, 3)
    hp, wp = _conv_out(h1, 3, 2, 1), _conv_out(w1, 3, 2, 1)
    h2, w2 = _conv_out(hp, 5, 2, 2), _conv_out(wp, 5, 2, 2)
    h3, w3 = _conv_out(h2, 3, 2, 1), _conv_out(w2, 3, 2, 1)
    h4, w4 = _conv_out(h3, 3, 2, 1), _conv_out(w3, 3, 2, 1)
    h5, w5 = _conv_out(h4, 3, 2, 1), _conv_out(w4, 3, 2, 1)
    if stage >= 32:
        return (detect.num_priors(h, w) * (4 if stage < 35 else 2),)
    fixed = {0: (h1, w1, 48), 1: (hp, wp, 48), 2: (h2, w2, 128), 3: (h3, w3, 128),
             28: (h3, w3, 128), 29: (h4, w4, 256), 30: (h4, w4, 128), 31: (h5, w5, 256)}
    if stage in fixed:
        return fixed[stage]
    return (h3, w3, {3: 24, 5: 24, 6: 32}.get((stage - 4) % 8, 128))         # inception: r1, r2, t3, else 128 channels


class FaceBoxes:
    """``FaceBoxes.FaceBoxes`` (FaceBoxes/FaceBoxes.py:46-143).  ``weights``: a state dict, a checkpoint path, or None for
    ``weights/FaceBoxesProd.pth`` next to this module (where the reference keeps it)."""

    def __init__(self, timer_flag: bool = False, weights=None, device=None):
        if weights is None:
            weights = os.path.join(os.path.dirname(os.path.realpath(__file__)), 'weights', 'FaceBoxesProd.pth')
        if isinstance(weights, (str, os.PathLike)):
            weights = torch.load(weights, map_location='cpu')
            if 'state_dict' in weights:
                weights = weights['state_dict']                                               # utils/functions.py:34-37
        self.net = FaceBoxesNet(weights, device)
        self.timer_flag = timer_flag

    def __call__(self, img_: np.ndarray):
        image = torch.from_numpy(np.ascontiguousarray(img_, dtype=np.uint8)).to(self.net.device)
        h, w = img_.shape[:2]
        scale, dsize = shrink_size(h, w)                                                      # FaceBoxes.py:62-79
        if scale != 1:                                                                        # cv2.resize, INTER_LINEAR
            image = crop_resize_device(image, [[0, 0, w, h]], dsize, INTER_LINEAR, planar=False)[0]
        im_h, im_w = int(image.shape[0]), int(image.shape[1])
        loc, conf = self.net.forward(image)
        dets, n = detect.decode_device(loc, conf, im_h, im_w, scale=float(scale))
        n_host = int(n.item())
        if n_host == 0:
            return []
        keep, n_keep = detect.nms_device(dets, detect.nms_threshold, _lib.NMS_CPU_NMS, n=n_host)
        kept = dets[keep[:int(n_keep.item())].long()][:detect.keep_top_k].cpu().numpy()
        return [[b[0], b[1], b[2], b[3], b[4]] for b in kept if b[4] > detect.vis_thres]

    def detect_images(self, images):
        """``[self(img) for img in images]`` for images of any sizes: ``images`` is a list of BGR uint8 (H,W,3) host arrays or
        CUDA tensors (or an :class:`~synergynet_b200.inference.ImagePack` a caller already uploaded).

        One upload of the packed bytes; per chunk of at most ``_lib.FB_MAX_FRAMES`` images one crop launch shrinks every
        image above 720 x 1080 to its own size on the device, then network, decode and NMS run over the whole chunk; the
        kept boxes and counts of every chunk come back in one host synchronisation at the end."""
        pack = pack_images(images, self.net.device)
        pending = []
        for a, b in chunk_ranges(len(pack), _lib.FB_MAX_FRAMES):
            sub = pack.slice(a, b)
            shrink = [shrink_size(h, w) for h, w in sub.sizes]
            big = [i for i, (scale, _) in enumerate(shrink) if scale != 1]
            net_in = sub
            if big:                                                                            # FaceBoxes.py:62-79
                shrunk = crop_resize_images_device(sub, big, [[0, 0, sub.sizes[i][1], sub.sizes[i][0]] for i in big],
                                                   [shrink[i][1] for i in big], INTER_LINEAR, planar=False)
                parts, at = [], 0
                for i in range(len(sub)):
                    if shrink[i][0] != 1:
                        ow, oh = shrink[i][1]
                        parts.append(shrunk[at:at + 3 * oh * ow])
                        at += 3 * oh * ow
                    else:
                        parts.append(sub.image(i).reshape(-1))
                net_in = ImagePack(torch.cat(parts), [(d[1], d[0]) for _, d in shrink])
            scales = [float(sc) for sc, _ in shrink]
            loc, conf, _ = self.net.forward_packed(net_in)
            dets, n = detect.decode_images_device(loc, conf, net_in.sizes, scales)
            pending.append(self._nms_to_host(dets, n))
        return self._boxes_of(pending)

    def _nms_to_host(self, dets, n):
        """NMS of every frame of a decoded chunk and the asynchronous copy of its first keep_top_k kept rows and counts."""
        keep, n_keep = detect.nms_batch_device(dets, n, detect.nms_threshold, _lib.NMS_CPU_NMS)
        # the first keep_top_k kept rows of every frame (entries past a frame's count are unwritten: clamped, never read)
        idx = keep[:, :detect.keep_top_k].long().clamp_(0, dets.shape[1] - 1)
        kept = torch.gather(dets, 1, idx[:, :, None].expand(-1, -1, 5))
        kept_host = torch.empty(kept.shape, dtype=kept.dtype, pin_memory=True)
        n_host = torch.empty(n_keep.shape, dtype=n_keep.dtype, pin_memory=True)
        kept_host.copy_(kept, non_blocking=True)
        n_host.copy_(n_keep, non_blocking=True)
        return kept_host, n_host

    def _boxes_of(self, pending):
        """One host synchronisation, then every frame's box list from the chunks' copies."""
        torch.cuda.current_stream(self.net.device).synchronize()
        out = []
        for kept_host, n_host in pending:
            kept_np, n_np = kept_host.numpy(), n_host.numpy()
            for i in range(kept_np.shape[0]):
                rows = kept_np[i, :min(int(n_np[i]), detect.keep_top_k)]
                out.append([[b[0], b[1], b[2], b[3], b[4]] for b in rows if b[4] > detect.vis_thres])
        return out

    def detect_batch(self, frames):
        """``__call__`` for N frames of one size: ``frames`` is a list / (N,H,W,3) array of BGR uint8 images, or the uint8
        (N,H,W,3) CUDA stack a caller already uploaded.  Returns N box lists, ``detect_batch(frames)[i]`` being exactly
        ``self(frames[i])`` (the > 720 x 1080 shrink, ``keep_top_k`` and ``vis_thres`` included).

        One upload of the stack; network, decode and NMS run over all frames of a chunk (at most ``_lib.FB_MAX_FRAMES``
        frames) per launch, the counts going from decode to NMS on the device; the kept boxes and their counts of every
        chunk come back in one host synchronisation at the end, whatever N is."""
        stack = stack_frames_device(frames, self.net.device)
        h, w = int(stack.shape[1]), int(stack.shape[2])
        scale, dsize = shrink_size(h, w)                                                      # FaceBoxes.py:62-79
        pending = []
        for a, b in chunk_ranges(int(stack.shape[0]), _lib.FB_MAX_FRAMES):
            images = stack[a:b]
            if scale != 1:                                                                    # cv2.resize, INTER_LINEAR
                images = crop_resize_frames_device(images, list(range(b - a)), [[0, 0, w, h]] * (b - a), dsize, INTER_LINEAR,
                                                   planar=False)
            im_h, im_w = int(images.shape[1]), int(images.shape[2])
            loc, conf = self.net.forward_batch(images)
            dets, n = detect.decode_batch_device(loc, conf, im_h, im_w, scale=float(scale))
            pending.append(self._nms_to_host(dets, n))
        return self._boxes_of(pending)
