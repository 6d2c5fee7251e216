"""Sim3DR on the H100: vertex normals, lighting and z-buffer rasterisation (SURVEY.md section 8 row f2).

Reference-shaped surface (``Sim3DR/Sim3DR.py:8-29``, ``Sim3DR/lighting.py:23-79``): ``get_normal``, ``rasterize``,
``RenderPipeline`` take and return numpy arrays like the reference's Cython module does.  Underneath sits
:class:`MeshRenderer`, which works on device tensors and on a whole BATCH of meshes per launch -- it reads the dense
vertices ``reconstruct_vertex_62(dense=True)`` / ``syn_reconstruct_image`` leave on the GPU in place (any strides), so
the 638 KB per face never visit the host.  All arithmetic runs in ``libsynergy_b200.so`` (``csrc/kernels_render.cuh``);
there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib


def _light_cfg(**kw) -> _lib.LightCfg:
    """Defaults of ``RenderPipeline.__init__`` (Sim3DR/lighting.py:24-32)."""
    v3 = lambda x: (C.c_float * 3)(*[float(t) for t in x])
    return _lib.LightCfg(float(kw.get('intensity_ambient', 0.3)), float(kw.get('intensity_directional', 0.6)),
                         float(kw.get('intensity_specular', 0.1)), v3(kw.get('color_ambient', (1, 1, 1))),
                         v3(kw.get('color_directional', (1, 1, 1))), v3(kw.get('light_pos', (0, 0, 5))),
                         v3(kw.get('view_pos', (0, 0, 5))), int(kw.get('specular_exp', 5)))


class MeshRenderer:
    """Batched renderer over one triangle list.

    ``triangles``: (ntri,3) integer array, 0-based (``utils/render.py:32-33``).  Vertex arguments are float32 CUDA
    tensors indexed ``v[b, i, k]`` = coordinate k of vertex i of mesh b with ANY strides: pass
    ``dense.transpose(1, 2)`` for the (B,3,N) output of the 3DMM stage (a view, nothing is copied).
    """

    def __init__(self, triangles, nver: int, device=None):
        self._lib = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError('synergynet_b200.Sim3DR needs a CUDA device (H100, sm_90a); there is no CPU fallback')
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        tri = np.ascontiguousarray(np.asarray(triangles), dtype=np.int32)
        if tri.ndim != 2 or tri.shape[1] != 3:
            raise ValueError('triangles must be (ntri, 3)')
        self.nver, self.ntri = int(nver), int(tri.shape[0])
        start = np.zeros(self.nver + 1, np.int32)
        lst = np.zeros(max(3 * self.ntri, 1), np.int32)
        _lib.check(self._lib.syn_mesh_incidence_host(tri.ctypes.data, self.ntri, self.nver, start.ctypes.data, lst.ctypes.data))
        self.tri = torch.from_numpy(tri).to(self.device)
        self._inc_start = torch.from_numpy(start).to(self.device)
        self._inc_tri = torch.from_numpy(lst).to(self.device)
        self.launches = 0

    # -- helpers ----------------------------------------------------------------------------------------------------------
    def _view(self, vertices: torch.Tensor):
        if vertices.dim() == 2:
            vertices = vertices.unsqueeze(0)
        if vertices.dtype != torch.float32 or vertices.device != self.device or vertices.dim() != 3 \
                or vertices.shape[1] != self.nver or vertices.shape[2] != 3:
            raise ValueError(f'vertices must be float32 (B,{self.nver},3) on {self.device}; got {tuple(vertices.shape)} '
                             f'{vertices.dtype} on {vertices.device}')
        sb, sv, sc = vertices.stride()
        if vertices.shape[0] == 1:
            sb = max(sb, 1)
        if min(sb, sv, sc) <= 0:
            raise ValueError('vertices must have positive strides (no expanded / flipped views)')
        return vertices, (vertices.data_ptr(), int(sb), int(sv), int(sc), int(vertices.shape[0]), self.nver)

    def normals(self, vertices: torch.Tensor) -> torch.Tensor:
        """``get_normal`` for every mesh: (B,nver,3) unit normals (NaN for a vertex no triangle touches, like the reference)."""
        v, view = self._view(vertices)
        b = view[4]
        ws = torch.empty((b, self.ntri, 3), dtype=torch.float32, device=self.device)
        out = torch.empty((b, self.nver, 3), dtype=torch.float32, device=self.device)
        _lib.launch(self.device, 'syn_mesh_normals', *view, self.tri.data_ptr(), self.ntri, self._inc_start.data_ptr(),
                    self._inc_tri.data_ptr(), ws.data_ptr(), out.data_ptr())
        self.launches += 2
        return out

    def colors(self, vertices: torch.Tensor, normals: torch.Tensor, cfg: Optional[_lib.LightCfg] = None,
               texture: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Per-vertex light of ``RenderPipeline.__call__``, times ``texture`` if given -- (nver,3) for every mesh, or
        (B,nver,3), one texture per mesh (``syn_mesh_lighting_textures``): (B,nver,3) in [0,1]."""
        v, view = self._view(vertices)
        b = view[4]
        cfg = cfg or _light_cfg()
        normals = normals.contiguous()
        if tuple(normals.shape) != (b, self.nver, 3) or normals.dtype != torch.float32 or normals.device != self.device:
            raise ValueError('normals must be float32 (B,nver,3) on the renderer device')
        stats = torch.empty((b, 6), dtype=torch.int32, device=self.device)
        out = torch.empty((b, self.nver, 3), dtype=torch.float32, device=self.device)
        if texture is not None and texture.dim() == 3:
            texture = texture.to(device=self.device, dtype=torch.float32).contiguous()
            if tuple(texture.shape) != (b, self.nver, 3):
                raise ValueError(f'texture must be (nver, 3) or (B, nver, 3) = ({b}, {self.nver}, 3), got {tuple(texture.shape)}')
            _lib.launch(self.device, 'syn_mesh_lighting_textures', *view, normals.data_ptr(), C.byref(cfg), texture.data_ptr(),
                        3 * self.nver, stats.data_ptr(), out.data_ptr())
            self.launches += 2
            return out
        tex_ptr = None
        if texture is not None:
            texture = texture.to(device=self.device, dtype=torch.float32).contiguous()
            if tuple(texture.shape) != (self.nver, 3):
                raise ValueError('texture must be (nver, 3)')
            tex_ptr = texture.data_ptr()
        _lib.launch(self.device, 'syn_mesh_lighting', *view, normals.data_ptr(), C.byref(cfg), tex_ptr, stats.data_ptr(),
                    out.data_ptr())
        self.launches += 2
        return out

    def rasterize(self, image: torch.Tensor, vertices: torch.Tensor, colors: torch.Tensor, reverse: bool = False,
                  return_depth: bool = False):
        """Draw the B meshes, in order, onto ``image`` (H,W,C) uint8 on the device, IN PLACE (alpha = 1)."""
        v, view = self._view(vertices)
        b = view[4]
        if image.dtype != torch.uint8 or image.dim() != 3 or image.device != self.device or not image.is_contiguous():
            raise ValueError('image must be a contiguous uint8 (H,W,C) tensor on the renderer device')
        h, w, c = (int(s) for s in image.shape)
        colors = colors.contiguous()
        if tuple(colors.shape) != (b, self.nver, c) or colors.dtype != torch.float32 or colors.device != self.device:
            raise ValueError(f'colors must be float32 (B,nver,{c}) on the renderer device')
        keys = torch.empty((b, h, w), dtype=torch.int64, device=self.device)
        depth = torch.empty((b, h, w), dtype=torch.float32, device=self.device) if return_depth else None
        _lib.launch(self.device, 'syn_rasterize', image.data_ptr(), h, w, c, *view, self.tri.data_ptr(), self.ntri, colors.data_ptr(),
                    1.0, 1 if reverse else 0, keys.data_ptr(), depth.data_ptr() if depth is not None else None)
        self.launches += 2
        return (image, depth) if return_depth else image

    def render(self, image: torch.Tensor, vertices: torch.Tensor, cfg: Optional[_lib.LightCfg] = None,
               texture: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``RenderPipeline.__call__`` for a batch of meshes drawn one after the other onto ``image`` (in place)."""
        nrm = self.normals(vertices)
        return self.rasterize(image, vertices, self.colors(vertices, nrm, cfg, texture))

    # -- the frame axis ----------------------------------------------------------------------------------------------------
    @staticmethod
    def _mesh_start(counts, n_frames: int) -> np.ndarray:
        counts = [int(c) for c in counts]
        if len(counts) != n_frames or min(counts, default=0) < 0:
            raise ValueError(f'counts must give a non-negative mesh count for each of the {n_frames} frames, got {counts}')
        return np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)

    def plan_frames(self, vertices: torch.Tensor, counts, height: int, width: int):
        """Pixel boxes (M,4) int32 ``x0, y0, x1, y1`` of the M meshes on a ``height`` x ``width`` frame and the key offsets
        (M+1) int64 of :meth:`rasterize_frames` (``syn_render_frames_plan``).  ``counts[f]`` meshes belong to frame f."""
        v, view = self._view(vertices)
        m = view[4]
        start = self._mesh_start(counts, len(counts))
        boxes = torch.empty((m, 4), dtype=torch.int32, device=self.device)
        key_off = torch.empty(m + 1, dtype=torch.int64, device=self.device)
        _lib.launch(self.device, 'syn_render_frames_plan', *view, self.tri.data_ptr(), self.ntri, start.ctypes.data, len(counts),
                    int(height), int(width), boxes.data_ptr(), key_off.data_ptr())
        self.launches += 2
        return boxes, key_off

    def rasterize_frames(self, frames: torch.Tensor, vertices: torch.Tensor, colors: torch.Tensor, counts,
                         out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Solid overlays of a frame stack: ``frames`` (N,H,W,C) uint8, frame f's meshes are the next ``counts[f]`` of the
        M meshes of ``vertices`` / ``colors`` (M,nver,C), drawn in order as :meth:`rasterize` draws them onto one image.
        Returns ``out`` (a new stack if None; ``out=frames`` draws in place).  One host synchronisation: the key count."""
        v, view = self._view(vertices)
        m = view[4]
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.device != self.device or not frames.is_contiguous():
            raise ValueError('frames must be a contiguous uint8 (N,H,W,C) tensor on the renderer device')
        n, h, w, c = (int(s) for s in frames.shape)
        colors = colors.contiguous()
        if colors.dim() != 3 or tuple(colors.shape[:2]) != (m, self.nver) or colors.dtype != torch.float32 or colors.device != self.device:
            raise ValueError(f'colors must be float32 (M,nver,C) on the renderer device; got {tuple(colors.shape)}')
        if out is None:
            out = torch.empty_like(frames)
        elif out.shape != frames.shape or out.dtype != torch.uint8 or out.device != self.device or not out.is_contiguous():
            raise ValueError('out must be a contiguous uint8 tensor shaped like frames')
        start = self._mesh_start(counts, n)
        boxes, key_off = self.plan_frames(v, counts, h, w)
        n_keys = int(key_off[m].item())                                   # the stage's one host synchronisation
        keys = torch.empty(max(n_keys, 1), dtype=torch.int64, device=self.device)
        self.last_key_count = n_keys
        start_dev = torch.from_numpy(start).to(self.device)
        _lib.launch(self.device, 'syn_rasterize_frames', frames.data_ptr(), out.data_ptr(), n, h, w, c, *view, self.tri.data_ptr(),
                    self.ntri, colors.data_ptr(), int(colors.shape[2]), start.ctypes.data, start_dev.data_ptr(), boxes.data_ptr(),
                    key_off.data_ptr(), n_keys, keys.data_ptr(), keys.numel())
        self.launches += 2
        return out

    def render_frames(self, frames_dev: torch.Tensor, vertices: torch.Tensor, counts, cfg: Optional[_lib.LightCfg] = None,
                      texture: Optional[torch.Tensor] = None, alpha: float = 0.6):
        """``utils/render.py:38-45`` for every frame of a stack at once: frame f's ``counts[f]`` meshes (the next ones of
        ``vertices`` (M,nver,3), any strides: ``reconstruct_image(...).transpose(1, 2)``) are lit and drawn onto a copy of
        it, which is then blended with it as ``cv2.addWeighted(frame, 1 - alpha, solid, alpha, 0)``.  Returns the device
        stacks ``(blended, solid)``, each frame's bytes those of :func:`render` on that frame alone."""
        if sum(int(c) for c in counts) == 0:
            self._mesh_start(counts, int(frames_dev.shape[0]))
            solid = frames_dev.clone()
        else:
            col = self.colors(vertices, self.normals(vertices), cfg, texture)
            solid = self.rasterize_frames(frames_dev, vertices, col, counts)
        return add_weighted(frames_dev, solid, alpha), solid

    # -- the image list: images of any sizes -----------------------------------------------------------------------------
    def _image_axis(self, pack, counts):
        """Host and device copies of the image table (n,3) int64 (offset, h, w) and of mesh_start (n+1) int32 of an
        :class:`~synergynet_b200.inference.ImagePack`: ``(table, start, device buffer, table_dev ptr, start_dev ptr)``.
        One upload carries both device copies."""
        from .inference import ImagePack
        if not isinstance(pack, ImagePack) or pack.data.device != self.device or pack.data.dtype != torch.uint8 \
                or not pack.data.is_contiguous():
            raise ValueError('images must be an ImagePack of uint8 bytes on the renderer device')
        n = len(pack)
        start = self._mesh_start(counts, n)
        table = np.array([[o, h, w] for o, (h, w) in zip(pack.offsets[:-1], pack.sizes)], np.int64).reshape(n, 3)
        buf = np.zeros(3 * n + (n + 2) // 2, np.int64)
        buf[:3 * n] = table.reshape(-1)
        buf[3 * n:].view(np.int32)[:n + 1] = start
        dev = torch.from_numpy(buf).to(self.device)
        return table, start, dev, dev.data_ptr(), dev[3 * n:].data_ptr()

    def plan_images(self, pack, vertices: torch.Tensor, counts):
        """:meth:`plan_frames` for the images of an ImagePack (``syn_render_images_plan``): each mesh's box is clamped to
        its own image.  ``counts[i]`` meshes belong to image i."""
        return self._plan_images(pack, vertices, self._image_axis(pack, counts))

    def _plan_images(self, pack, vertices, axis):
        v, view = self._view(vertices)
        m = view[4]
        table, start, _keep, table_dev, start_dev = axis
        boxes = torch.empty((m, 4), dtype=torch.int32, device=self.device)
        key_off = torch.empty(m + 1, dtype=torch.int64, device=self.device)
        _lib.launch(self.device, 'syn_render_images_plan', *view, self.tri.data_ptr(), self.ntri, start.ctypes.data, start_dev,
                    table.ctypes.data, table_dev, len(pack), pack.data.numel(), 3, boxes.data_ptr(), key_off.data_ptr())
        self.launches += 2
        return boxes, key_off

    def rasterize_images(self, pack, vertices: torch.Tensor, colors: torch.Tensor, counts, out=None):
        """:meth:`rasterize_frames` for the images of an :class:`~synergynet_b200.inference.ImagePack`: image i's meshes
        are the next ``counts[i]`` of ``vertices`` / ``colors`` (M,nver,3), drawn in order, each clamped to its own image.
        Returns ``out``, an ImagePack of the same sizes (a new one if None; ``out=pack`` draws in place).  One host
        synchronisation: the key count."""
        from .inference import ImagePack
        v, view = self._view(vertices)
        m = view[4]
        colors = colors.contiguous()
        if colors.dim() != 3 or tuple(colors.shape[:2]) != (m, self.nver) or colors.dtype != torch.float32 or colors.device != self.device:
            raise ValueError(f'colors must be float32 (M,nver,C) on the renderer device; got {tuple(colors.shape)}')
        if not isinstance(pack, ImagePack):
            raise ValueError('images must be an ImagePack')
        if out is None:
            out = ImagePack(torch.empty_like(pack.data), pack.sizes)
        elif not isinstance(out, ImagePack) or out.sizes != pack.sizes or out.data.dtype != torch.uint8 \
                or out.data.device != self.device or not out.data.is_contiguous():
            raise ValueError('out must be an ImagePack of the sizes of the images, on the renderer device')
        axis = self._image_axis(pack, counts)
        table, start, _keep, table_dev, start_dev = axis
        boxes, key_off = self._plan_images(pack, v, axis)
        n_keys = int(key_off[m].item())                                   # the stage's one host synchronisation
        keys = torch.empty(max(n_keys, 1), dtype=torch.int64, device=self.device)
        self.last_key_count = n_keys
        _lib.launch(self.device, 'syn_rasterize_images', pack.data.data_ptr(), out.data.data_ptr(), pack.data.numel(), table.ctypes.data,
                    table_dev, len(pack), 3, *view, self.tri.data_ptr(), self.ntri, colors.data_ptr(), int(colors.shape[2]),
                    start.ctypes.data, start_dev, boxes.data_ptr(), key_off.data_ptr(), n_keys, keys.data_ptr(), keys.numel())
        self.launches += 2
        return out

    def render_images(self, pack, vertices: torch.Tensor, counts, cfg: Optional[_lib.LightCfg] = None,
                      texture: Optional[torch.Tensor] = None, alpha: float = 0.6):
        """:meth:`render_frames` for the images of an ImagePack: ``(blended, solid)`` ImagePacks, image i's bytes those
        of :func:`render` on that image alone with its ``counts[i]`` meshes."""
        from .inference import ImagePack
        if sum(int(c) for c in counts) == 0:
            self._mesh_start(counts, len(pack))
            solid = ImagePack(pack.data.clone(), pack.sizes)
        else:
            col = self.colors(vertices, self.normals(vertices), cfg, texture)
            solid = self.rasterize_images(pack, vertices, col, counts)
        return ImagePack(add_weighted(pack.data, solid.data, alpha), pack.sizes), solid


def add_weighted(a: torch.Tensor, b: torch.Tensor, alpha: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``cv2.addWeighted(a, 1 - alpha, b, alpha, 0)`` of two uint8 CUDA tensors of one shape, byte for byte
    (``syn_add_weighted_u8``).  ``out`` may be ``a`` or ``b``."""
    if a.dtype != torch.uint8 or b.dtype != torch.uint8 or a.shape != b.shape or not a.is_cuda or a.device != b.device:
        raise ValueError('add_weighted takes two uint8 CUDA tensors of one shape on one device')
    a, b = a.contiguous(), b.contiguous()
    out = torch.empty_like(a) if out is None else out
    if out.shape != a.shape or out.dtype != torch.uint8 or out.device != a.device or not out.is_contiguous():
        raise ValueError('out must be a contiguous uint8 tensor shaped like the inputs')
    _lib.launch(a.device, 'syn_add_weighted_u8', a.data_ptr(), b.data_ptr(), float(alpha), out.data_ptr(), a.numel())
    return out


_renderers = {}


def _renderer_for(triangles: np.ndarray, nver: int) -> MeshRenderer:
    if not torch.cuda.is_available():
        raise RuntimeError('synergynet_b200.Sim3DR needs a CUDA device (H100, sm_90a); there is no CPU fallback')
    tri = np.ascontiguousarray(triangles, dtype=np.int32)
    key = (hash(tri.tobytes()), tri.shape, int(nver), torch.cuda.current_device())
    r = _renderers.get(key)
    if r is None:
        if len(_renderers) > 8:
            _renderers.clear()
        r = _renderers[key] = MeshRenderer(tri, nver)
    return r


def _verts_dev(vertices: np.ndarray, r: MeshRenderer) -> torch.Tensor:
    v = np.ascontiguousarray(vertices, dtype=np.float32)
    if v.ndim != 2 or v.shape[1] != 3:
        raise ValueError('vertices must be (nver, 3)')
    return torch.from_numpy(v).to(r.device).unsqueeze(0)


def get_normal(vertices: np.ndarray, triangles: np.ndarray) -> np.ndarray:
    """``Sim3DR.get_normal`` (Sim3DR/Sim3DR.py:8-11): (nver,3) float32 vertices, (ntri,3) int32 triangles -> (nver,3)."""
    r = _renderer_for(triangles, vertices.shape[0])
    return r.normals(_verts_dev(vertices, r))[0].cpu().numpy()


def rasterize(vertices, triangles, colors, bg=None, height=None, width=None, channel=None, reverse=False):
    """``Sim3DR.rasterize`` (Sim3DR/Sim3DR.py:14-29).  ``bg`` (H,W,C) uint8 is drawn into and returned, as the reference's
    C routine writes through the array it is given.  Without ``bg`` the reference builds a float32 canvas that its own
    ``unsigned char`` Cython signature then rejects; here that case starts from a black uint8 canvas."""
    if bg is not None:
        height, width, channel = bg.shape
    else:
        assert height is not None and width is not None and channel is not None
        bg = np.zeros((height, width, channel), dtype=np.uint8)
    if bg.dtype != np.uint8:
        raise ValueError("Buffer dtype mismatch, expected 'unsigned char'")       # what the reference's Cython layer raises
    colors = np.ascontiguousarray(colors, dtype=np.float32)
    r = _renderer_for(triangles, vertices.shape[0])
    img = torch.from_numpy(np.ascontiguousarray(bg)).to(r.device)
    r.rasterize(img, _verts_dev(vertices, r), torch.from_numpy(colors).to(r.device).unsqueeze(0), reverse=reverse)
    out = img.cpu().numpy()
    if bg.flags.writeable and bg.flags.c_contiguous:
        bg[...] = out
        return bg
    return out


def convert_type(obj):
    if isinstance(obj, (tuple, list)):
        return np.array(obj, dtype=np.float32)[None, :]
    return obj


class RenderPipeline(object):
    """``Sim3DR.RenderPipeline`` (Sim3DR/lighting.py:23-79): same constructor keywords and call signature."""

    def __init__(self, **kwargs):
        self._kw = dict(kwargs)
        self.light_pos = convert_type(kwargs.get('light_pos', (0, 0, 5)))

    def update_light_pos(self, light_pos):
        self.light_pos = convert_type(light_pos)

    def _cfg(self) -> _lib.LightCfg:
        kw = dict(self._kw)
        kw['light_pos'] = tuple(np.asarray(self.light_pos, np.float32).reshape(-1))
        return _light_cfg(**kw)

    def __call__(self, vertices, triangles, bg, texture=None):
        r = _renderer_for(triangles, vertices.shape[0])
        v = _verts_dev(vertices, r)
        tex = None if texture is None else torch.from_numpy(np.ascontiguousarray(texture, dtype=np.float32))
        col = r.colors(v, r.normals(v), self._cfg(), tex)
        if texture is not None and isinstance(texture, np.ndarray) and texture.flags.writeable:
            texture[...] = col[0].cpu().numpy()                                    # `texture *= light` is in place (:73)
        if bg.dtype != np.uint8:
            raise ValueError("Buffer dtype mismatch, expected 'unsigned char'")
        img = torch.from_numpy(np.ascontiguousarray(bg)).to(r.device)
        r.rasterize(img, v, col)
        out = img.cpu().numpy()
        if bg.flags.writeable and bg.flags.c_contiguous:
            bg[...] = out
            return bg
        return out


def render(img: np.ndarray, ver_lst, tri, alpha: float = 0.6, wfp=None, tex=None, cfg: Optional[dict] = None):
    """``utils/render.py:31-53`` as one batched call: every (3,N) vertex array of ``ver_lst`` is lit and drawn, in order,
    onto a copy of ``img`` (the loop :41-45 becomes one launch sequence over the batch), then blended with
    ``cv2.addWeighted(img, 1 - alpha, overlap, alpha, 0)``.  ``tri``: (ntri,3) 0-based triangles (the reference re-reads
    ``3dmm_data/tri.mat`` on every call).  Returns ``(blended, overlap)``."""
    import cv2
    from .inference import RENDER_CFG
    ver = np.stack([np.asarray(v, dtype=np.float32) for v in ver_lst])             # (B,3,N)
    r = _renderer_for(tri, ver.shape[2])
    v = torch.from_numpy(ver).to(r.device).transpose(1, 2)                          # strided view, no transpose copy
    canvas = torch.from_numpy(np.ascontiguousarray(img)).to(r.device)
    texture = None if tex is None else torch.from_numpy(np.ascontiguousarray(tex, dtype=np.float32))
    r.render(canvas, v, _light_cfg(**(cfg or RENDER_CFG)), texture)
    overlap = canvas.cpu().numpy()
    res = cv2.addWeighted(img, 1 - alpha, overlap, alpha, 0)
    if wfp is not None:
        cv2.imwrite(wfp[:-4] + '_solid' + '.png', overlap)
        cv2.imwrite(wfp, res)
    return res, overlap


def render_batch(frames, ver_lsts, tri, alpha: float = 0.6, wfps=None, tex=None, cfg: Optional[dict] = None):
    """:func:`render` for N equally sized frames in one pass: entry i of the returned list is the ``(blended, overlap)``
    pair ``render(frames[i], ver_lsts[i], tri, alpha, wfps[i], tex, cfg)`` returns, bit for bit.  One upload of the frames
    and of all meshes, one normals / lighting / rasterisation / blend launch sequence for all of them, one download of
    each result stack.  A frame without a mesh gets ``overlap = frame`` and ``blended = cv2.addWeighted(frame, 1 - alpha,
    frame, alpha, 0)``, as the reference's ``render(img, [], ...)`` computes.  ``wfps``: None, or one path (or None) per
    frame, written as :func:`render` writes them."""
    import cv2
    from .inference import RENDER_CFG, stack_frames_host
    stack = stack_frames_host(frames)
    n = stack.shape[0]
    if len(ver_lsts) != n or (wfps is not None and len(wfps) != n):
        raise ValueError(f'{len(ver_lsts)} mesh lists and {"no" if wfps is None else len(wfps)} paths for {n} frames')
    counts = [len(v) for v in ver_lsts]
    meshes = [np.asarray(v, dtype=np.float32) for vl in ver_lsts for v in vl]
    if not torch.cuda.is_available():
        raise RuntimeError('synergynet_b200.Sim3DR needs a CUDA device (H100, sm_90a); there is no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device())
    frames_dev = torch.from_numpy(stack).to(dev)
    if meshes:
        ver = np.stack(meshes)                                                      # (M,3,N)
        r = _renderer_for(tri, ver.shape[2])
        v = torch.from_numpy(ver).to(r.device).transpose(1, 2)
        texture = None if tex is None else torch.from_numpy(np.ascontiguousarray(tex, dtype=np.float32))
        blended, solid = r.render_frames(frames_dev, v, counts, _light_cfg(**(cfg or RENDER_CFG)), texture, alpha)
    else:
        solid = frames_dev
        blended = add_weighted(frames_dev, solid, alpha)
    blended, solid = blended.cpu().numpy(), solid.cpu().numpy()
    out = []
    for i in range(n):
        res, overlap = blended[i], solid[i]
        if wfps is not None and wfps[i] is not None:
            cv2.imwrite(wfps[i][:-4] + '_solid' + '.png', overlap)
            cv2.imwrite(wfps[i], res)
        out.append((res, overlap))
    return out


def render_images(images, ver_lsts, tri, alpha: float = 0.6, wfps=None, tex=None, cfg: Optional[dict] = None):
    """:func:`render_batch` for N images of any sizes (a list of (h_i,w_i,3) uint8 arrays): entry i of the returned list is
    the ``(blended, overlap)`` pair ``render(images[i], ver_lsts[i], tri, alpha, wfps[i], tex, cfg)`` returns, bit for
    bit.  One upload of the packed images and of all meshes, one normals / lighting / rasterisation / blend launch
    sequence for all of them, one download of each result pack.  An image without a mesh gets ``overlap = image`` and
    ``blended = cv2.addWeighted(image, 1 - alpha, image, alpha, 0)``, as :func:`render_batch` gives a frame without one."""
    import cv2
    from .inference import RENDER_CFG, pack_images
    images = [np.asarray(im) for im in images]
    n = len(images)
    if not n:
        raise ValueError('no images: an image list needs at least one image')
    if len(ver_lsts) != n or (wfps is not None and len(wfps) != n):
        raise ValueError(f'{len(ver_lsts)} mesh lists and {"no" if wfps is None else len(wfps)} paths for {n} images')
    for im in images:
        if im.ndim != 3 or im.shape[2] != 3 or im.shape[0] < 1 or im.shape[1] < 1:
            raise ValueError(f'every image must be (H,W,3) with H, W >= 1, got {tuple(im.shape)}')
    counts = [len(v) for v in ver_lsts]
    meshes = [np.asarray(v, dtype=np.float32) for vl in ver_lsts for v in vl]
    if not torch.cuda.is_available():
        raise RuntimeError('synergynet_b200.Sim3DR needs a CUDA device (H100, sm_90a); there is no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device())
    pack = pack_images(images, dev)
    if meshes:
        ver = np.stack(meshes)                                                      # (M,3,N)
        r = _renderer_for(tri, ver.shape[2])
        v = torch.from_numpy(ver).to(r.device).transpose(1, 2)
        texture = None if tex is None else torch.from_numpy(np.ascontiguousarray(tex, dtype=np.float32))
        blended, solid = r.render_images(pack, v, counts, _light_cfg(**(cfg or RENDER_CFG)), texture, alpha)
        blended, solid = blended.data, solid.data
    else:
        solid = pack.data
        blended = add_weighted(pack.data, solid, alpha)
    blended, solid = blended.cpu().numpy(), solid.cpu().numpy()
    out = []
    for i, (h, w) in enumerate(pack.sizes):
        a, b = pack.offsets[i], pack.offsets[i + 1]
        res, overlap = blended[a:b].reshape(h, w, 3), solid[a:b].reshape(h, w, 3)
        if wfps is not None and wfps[i] is not None:
            cv2.imwrite(wfps[i][:-4] + '_solid' + '.png', overlap)
            cv2.imwrite(wfps[i], res)
        out.append((res, overlap))
    return out
