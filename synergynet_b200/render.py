"""``utils/render.py`` of the reference on the H100: ``render(img, ver_lst, alpha, wfp, tex, connectivity)`` with the
reference's signature and return value (utils/render.py:31-53).  The triangle list comes from the same place as the
reference's (``3dmm_data/tri.mat`` through the parameter pack, 1-based in the file) unless ``connectivity`` is given; the
per-face loop :41-45 is one batched call of :func:`synergynet_b200.Sim3DR.render` (normals, lighting, z-buffer on the
device; ``cv2.addWeighted`` and the PNG writes stay on the host as in the reference)."""
from __future__ import annotations

import numpy as np

from . import Sim3DR
from .inference import RENDER_CFG
from .params import get_param_pack

cfg = dict(RENDER_CFG)                                   # utils/render.py:18-27
render_app = Sim3DR.RenderPipeline(**cfg)                # :29 (per-face callable, same object name)


def _to_ctype(arr):
    return arr if arr.flags.c_contiguous else arr.copy(order='C')


def _triangles(connectivity):
    if connectivity is not None:
        return _to_ctype(np.asarray(connectivity).T).astype(np.int32)                 # :35-36
    pack_tri = get_param_pack().tri
    if pack_tri is None:
        raise RuntimeError('Missing data: 3dmm_data/tri.mat')                        # the reference's loadmat would raise here
    return _to_ctype((np.asarray(pack_tri) - 1).T).astype(np.int32)                  # :32-33


def render(img, ver_lst, alpha=0.6, wfp=None, tex=None, connectivity=None):
    res, _overlap = Sim3DR.render(img, ver_lst, _triangles(connectivity), alpha=alpha, wfp=wfp, tex=tex, cfg=cfg)
    if wfp is not None:
        print(f'Save mesh result to {wfp}')
    return res


def render_batch(imgs, ver_lsts, alpha=0.6, wfps=None, tex=None, connectivity=None):
    """:func:`render` for N equally sized frames in one pass (:func:`synergynet_b200.Sim3DR.render_batch`): returns the
    list of blended images, entry i being ``render(imgs[i], ver_lsts[i], alpha, wfps[i], tex, connectivity)``."""
    out = Sim3DR.render_batch(imgs, ver_lsts, _triangles(connectivity), alpha=alpha, wfps=wfps, tex=tex, cfg=cfg)
    for wfp in wfps or []:
        if wfp is not None:
            print(f'Save mesh result to {wfp}')
    return [res for res, _overlap in out]


def render_images(imgs, ver_lsts, alpha=0.6, wfps=None, tex=None, connectivity=None):
    """:func:`render` for N images of any sizes in one pass (:func:`synergynet_b200.Sim3DR.render_images`): returns the
    list of blended images, entry i being ``render(imgs[i], ver_lsts[i], alpha, wfps[i], tex, connectivity)``."""
    out = Sim3DR.render_images(imgs, ver_lsts, _triangles(connectivity), alpha=alpha, wfps=wfps, tex=tex, cfg=cfg)
    for wfp in wfps or []:
        if wfp is not None:
            print(f'Save mesh result to {wfp}')
    return [res for res, _overlap in out]
