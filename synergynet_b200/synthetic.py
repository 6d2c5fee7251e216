"""Seeded synthetic stand-ins for the assets the reference downloads at install time.

The reference needs ``3dmm_data/`` (BFM basis, whitening statistics, triangles), a trained
checkpoint and AFLW2000 crops (reference ``README.md:54-59``); none of them ship with it and
this project has no network.  Everything here is a deterministic function of a seed so that the
container that generates golden vectors and the GPU box that checks them see the same bytes.

File names / shapes follow what ``utils/params.py:13-35`` and ``model_building.py:68`` load.
Scaling follows SURVEY.md section 8(d) ("AFLW2000-style"): landmarks fall in the 120x120 crop.
"""
from __future__ import annotations

import os
import pickle

import numpy as np
import torch

NVER = 53215          # BFM vertex count used by the reference (model_building.py:125)
NTRI = 105840
N_SHP, N_EXP = 40, 10
STD_SIZE = 120


def _rot(yaw: float, pitch: float, roll: float) -> np.ndarray:
    cy, sy = np.cos(yaw), np.sin(yaw)
    cp, sp = np.cos(pitch), np.sin(pitch)
    cr, sr = np.cos(roll), np.sin(roll)
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rx = np.array([[1, 0, 0], [0, cp, -sp], [0, sp, cp]])
    rz = np.array([[cr, -sr, 0], [sr, cr, 0], [0, 0, 1]])
    return rz @ rx @ ry


def make_3dmm(seed: int = 0, nver: int = NVER) -> dict:
    """Synthetic morphable model with the reference's array shapes and dtypes."""
    rng = np.random.default_rng(seed)
    # mean shape: points on an ellipsoid of semi-axes ~(7e4, 9e4, 6e4) model units
    d = rng.standard_normal((nver, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    mean_xyz = d * np.array([7.0e4, 9.0e4, 6.0e4])
    u_shp = mean_xyz.reshape(-1, 1).astype(np.float32)                 # (3N,1) xyz interleaved
    u_exp = (rng.standard_normal((3 * nver, 1)) * 2.0e2).astype(np.float32)
    w_shp = rng.standard_normal((3 * nver, N_SHP)).astype(np.float32)
    w_exp = rng.standard_normal((3 * nver, N_EXP)).astype(np.float32)

    kv = np.sort(rng.choice(nver, 68, replace=False))
    keypoints = np.stack([3 * kv, 3 * kv + 1, 3 * kv + 2], 1).reshape(-1).astype(np.int64)

    mean = np.zeros(62, np.float32)
    std = np.zeros(62, np.float32)
    s = 5.0e-4
    cam = np.concatenate([s * _rot(0.3, -0.1, 0.05), np.array([[60.0], [60.0], [0.0]])], 1)
    mean[:12] = cam.reshape(-1)
    std12 = np.full((3, 4), 6.0e-5)
    std12[:, 3] = 4.0
    std[:12] = std12.reshape(-1)
    decay_s = 1.0 / np.sqrt(1.0 + np.arange(N_SHP))
    decay_e = 1.0 / np.sqrt(1.0 + np.arange(N_EXP))
    mean[12:52] = rng.standard_normal(N_SHP) * 300.0 * decay_s
    std[12:52] = 900.0 * decay_s
    mean[52:62] = rng.standard_normal(N_EXP) * 150.0 * decay_e
    std[52:62] = 400.0 * decay_e

    tri = rng.integers(1, nver + 1, (3, NTRI)).astype(np.int32)        # 1-based like tri.mat
    return dict(keypoints=keypoints, w_shp=w_shp, w_exp=w_exp, u_shp=u_shp, u_exp=u_exp,
                param_mean=mean, param_std=std, tri=tri)


def write_3dmm_dir(path: str, pack: dict) -> None:
    """Write ``pack`` with the file names ``utils/params.py:13-25`` reads."""
    import scipy.io as sio
    os.makedirs(path, exist_ok=True)
    np.save(os.path.join(path, 'keypoints_sim.npy'), pack['keypoints'])
    np.save(os.path.join(path, 'w_shp_sim.npy'), pack['w_shp'])
    np.save(os.path.join(path, 'w_exp_sim.npy'), pack['w_exp'])
    np.save(os.path.join(path, 'u_shp.npy'), pack['u_shp'])
    np.save(os.path.join(path, 'u_exp.npy'), pack['u_exp'])
    with open(os.path.join(path, 'param_whitening.pkl'), 'wb') as f:
        pickle.dump({'param_mean': pack['param_mean'], 'param_std': pack['param_std']}, f)
    sio.savemat(os.path.join(path, 'tri.mat'), {'tri': pack['tri']})


def make_crops_u8(batch: int, seed: int = 0) -> torch.Tensor:
    """(B,3,120,120) uint8 pixels; BASELINE.md section 3 synthetic input recipe."""
    g = torch.Generator().manual_seed(1000 + seed)
    return torch.randint(0, 256, (batch, 3, STD_SIZE, STD_SIZE), generator=g, dtype=torch.uint8)


def make_structured_crops_u8(batch: int, seed: int = 0) -> torch.Tensor:
    """(B,3,120,120) uint8 crops with low-frequency structure (ramps, a sinusoid, a blob) plus
    noise, so that different faces give visibly different network outputs (pure uniform noise
    is statistically identical from crop to crop once it has been average-pooled)."""
    g = torch.Generator().manual_seed(4000 + seed)
    lin = torch.linspace(-1.0, 1.0, STD_SIZE, dtype=torch.float64)
    yy, xx = torch.meshgrid(lin, lin, indexing='ij')
    out = torch.empty((batch, 3, STD_SIZE, STD_SIZE), dtype=torch.uint8)
    for b in range(batch):
        img = torch.zeros((3, STD_SIZE, STD_SIZE), dtype=torch.float64)
        for c in range(3):
            a = torch.randn(5, generator=g, dtype=torch.float64)
            img[c] = 128 + 60 * (a[0] * xx + a[1] * yy) + 50 * torch.sin(3 * a[2] * xx + 2 * a[3] * yy + a[4])
        q = torch.rand(3, generator=g, dtype=torch.float64)
        blob = torch.exp(-((xx - (q[0] * 1.2 - 0.6)) ** 2 + (yy - (q[1] * 1.2 - 0.6)) ** 2) / (0.05 + 0.2 * q[2]))
        img += 80 * blob * torch.randn((3, 1, 1), generator=g, dtype=torch.float64)
        img += 12 * torch.randn((3, STD_SIZE, STD_SIZE), generator=g, dtype=torch.float64)
        out[b] = img.clamp(0, 255).round().to(torch.uint8)
    return out


def normalize_crops(u8: torch.Tensor) -> torch.Tensor:
    """``(img - 127.5) / 128`` as in synergy3DMM.py:192 / benchmark.py:116."""
    return (u8.to(torch.float32) - 127.5) / 128.0


def make_inputs(batch: int, seed: int = 0) -> torch.Tensor:
    return normalize_crops(make_crops_u8(batch, seed))


@torch.no_grad()
def randomize_batchnorm_(module: torch.nn.Module, seed: int = 0) -> None:
    """Non-trivial BN statistics so that folding BN into the convs is actually exercised
    (the default init is the identity, mobilenetv2_backbone.py:166-168)."""
    g = torch.Generator().manual_seed(2000 + seed)
    for m in module.modules():
        if isinstance(m, (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d)):
            n = m.num_features
            m.weight.copy_(torch.rand(n, generator=g) * 0.5 + 0.75)
            m.bias.copy_(torch.randn(n, generator=g) * 0.1)
            m.running_mean.copy_(torch.randn(n, generator=g) * 0.1)
            m.running_var.copy_(torch.rand(n, generator=g) * 0.5 + 0.75)


@torch.no_grad()
def seeded_init_(module: torch.nn.Module, seed: int = 0) -> None:
    """Same distributions as the reference initialiser (mobilenetv2_backbone.py:161-171:
    kaiming-normal fan_out convs, normal linears) from a private generator; linears are
    N(0, 0.05) with N(0, 0.05) biases so the 62 outputs are O(1) and vary from face to face."""
    g = torch.Generator().manual_seed(3000 + seed)
    for m in module.modules():
        if isinstance(m, (torch.nn.Conv2d, torch.nn.Conv1d)):
            fan_out = m.weight.shape[0] * m.weight[0][0].numel()
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (2.0 / fan_out) ** 0.5)
            if m.bias is not None:
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.01)
        elif isinstance(m, torch.nn.Linear):
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) * 0.05)
            m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.05)


# ---- meshes for the Sim3DR stage (SURVEY.md section 8 row f2) ----------------------------------------------------------------
RENDER_ROWS, RENDER_COLS = 145, 367          # 145 * 367 = 53 215 = NVER vertices, 2 * 144 * 366 = 105 408 triangles


def make_render_topology(rows: int = RENDER_ROWS, cols: int = RENDER_COLS) -> np.ndarray:
    """(ntri,3) int32, 0-based: two triangles per cell of a rows x cols vertex grid (the real ``tri.mat`` is an external
    download; the random triangles of ``make_3dmm`` span the whole face and are useless for rendering)."""
    idx = np.arange(rows * cols, dtype=np.int32).reshape(rows, cols)
    a, b, c, d = idx[:-1, :-1], idx[1:, :-1], idx[:-1, 1:], idx[1:, 1:]
    return np.ascontiguousarray(np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([b, d, c], -1).reshape(-1, 3)]))


def make_render_meshes(batch: int, height: int, width: int, seed: int = 0, rows: int = RENDER_ROWS, cols: int = RENDER_COLS,
                       size: float = 0.0) -> np.ndarray:
    """(B,3,rows*cols) float32 vertices in image coordinates, plane-major like the dense output of the 3DMM stage: a
    grid wrapped over 3/4 of an ellipsoid (so that parts of every mesh face away and occlude each other), randomly
    posed, ``size`` pixels across (default: a third of the shorter image side), scattered over the image."""
    rng = np.random.default_rng(7000 + seed)
    size = size or min(height, width) / 3.0
    th = np.linspace(-0.75 * np.pi, 0.75 * np.pi, cols)[None, :]
    ph = np.linspace(-0.42 * np.pi, 0.42 * np.pi, rows)[:, None]
    base = np.stack([np.cos(ph) * np.sin(th) * 0.8, np.sin(ph) * np.ones_like(th), np.cos(ph) * np.cos(th) * 0.7], 0).reshape(3, -1)
    out = np.empty((batch, 3, rows * cols), np.float32)
    for b in range(batch):
        bump = 1.0 + 0.03 * np.sin(7 * th + rng.uniform(0, 6)) * np.cos(5 * ph + rng.uniform(0, 6))
        r = _rot(rng.uniform(-0.6, 0.6), rng.uniform(-0.4, 0.4), rng.uniform(-0.3, 0.3))
        p = r @ (base * bump.reshape(1, -1)) * (size / 2.0) * rng.uniform(0.8, 1.2)
        p[0] += rng.uniform(0.25, 0.75) * width
        p[1] += rng.uniform(0.25, 0.75) * height
        out[b] = p
    return out


# ---- detector weights (SURVEY.md section 8 row f3) ---------------------------------------------------------------------------
def make_faceboxes_state_dict(seed: int = 0):
    """Seeded stand-in for ``FaceBoxes/weights/FaceBoxesProd.pth`` in the reference's key schema: He-scaled conv weights
    (activations keep O(1) magnitude through the 12-layer-deep paths), non-trivial BatchNorm statistics so that folding is
    exercised, small head weights so that the class scores spread over (0,1)."""
    from .faceboxes import layer_plan
    g = torch.Generator().manual_seed(9000 + seed)
    sd = {}
    for L in layer_plan():
        fan_in = L['cin'] * L['ksize'] ** 2
        shape = (L['cout'], L['cin'], L['ksize'], L['ksize'])
        n = L['name']
        if L['has_bn']:
            sd[f'{n}.conv.weight'] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
            sd[f'{n}.bn.weight'] = torch.rand(L['cout'], generator=g) * 0.5 + 0.75
            sd[f'{n}.bn.bias'] = torch.randn(L['cout'], generator=g) * 0.1
            sd[f'{n}.bn.running_mean'] = torch.randn(L['cout'], generator=g) * 0.1
            sd[f'{n}.bn.running_var'] = torch.rand(L['cout'], generator=g) * 0.5 + 0.75
            if n == 'conv1':        # pixels minus the channel means are O(60): the first BatchNorm brings activations to O(1)
                sd[f'{n}.bn.running_var'] *= 7000.0
                sd[f'{n}.bn.running_mean'] *= 80.0
            sd[f'{n}.bn.num_batches_tracked'] = torch.tensor(0, dtype=torch.long)
        else:
            sd[f'{n}.weight'] = torch.randn(shape, generator=g) * (0.6 / fan_in) ** 0.5
            sd[f'{n}.bias'] = torch.randn(L['cout'], generator=g) * 0.05
    return sd


def make_scene_u8(height: int, width: int, seed: int = 0) -> np.ndarray:
    """(H,W,3) uint8 BGR test image: smooth gradients, a few ellipses, noise."""
    rng = np.random.default_rng(8000 + seed)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float32)
    img = np.stack([90 + 60 * np.sin(xx / 37.0 + c) + 40 * np.cos(yy / 23.0 - c) for c in range(3)], -1)
    for _ in range(4):
        cy, cx, r = rng.uniform(0.2, 0.8) * height, rng.uniform(0.2, 0.8) * width, rng.uniform(0.08, 0.2) * min(height, width)
        inside = ((yy - cy) / (1.25 * r)) ** 2 + ((xx - cx) / r) ** 2 < 1
        img[inside] = img[inside] * 0.3 + rng.uniform(60, 220, 3)
    img += rng.normal(0, 5, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


# ---- the UV layout of the textured flows (artistic.py, uv_texture_realFaces.py) -----------------------------------------------
def make_uv_layout(seed: int = 0, nver: int = NVER, dtype=np.float32, keep_fraction: float = 0.75):
    """Seeded stand-ins for ``3dmm_data/BFM_UV.npy`` (nver, 2) in ``dtype``, ``keptInd.npy`` (sorted int64) and
    ``deletedTri.npy`` ((3, ntri) int64, 1-based over the kept vertices).  The UV values include 0, 1.0 (texel 255) and the
    neighbours of k/255 on both sides, where ``(uv * 255.0).astype(np.int32)`` changes; about one kept vertex in twenty is
    touched by no triangle (a NaN normal in the reference, never drawn)."""
    rng = np.random.default_rng(11000 + seed)
    uv = rng.uniform(0.0, 1.0, (nver, 2)).astype(dtype)
    k = rng.integers(0, 256, (nver, 2))
    edge = (k / 255.0).astype(dtype)
    pick = rng.integers(0, 4, (nver, 2))
    uv = np.where(pick == 0, np.nextafter(edge, dtype(2)), np.where(pick == 1, np.nextafter(edge, dtype(-1)), uv)).astype(dtype)
    uv = np.where(pick == 2, edge, uv).astype(dtype)
    uv[:4] = np.array([[0, 0], [1, 1], [0, 1], [1, 0]], dtype)
    uv = np.clip(uv, 0, 1).astype(dtype)
    keep = np.sort(rng.choice(nver, max(1, int(nver * keep_fraction)), replace=False)).astype(np.int64)
    n_keep = keep.size
    used = rng.permutation(n_keep)[: max(3, n_keep - n_keep // 20)]
    ntri = 2 * n_keep
    tri = used[rng.integers(0, used.size, (3, ntri))].astype(np.int64) + 1
    return uv, keep, tri


def make_uv_map(height: int, width: int, seed: int = 0, channels: int = 3) -> np.ndarray:
    """(h, w, channels) uint8 UV map: smooth colour ramps plus noise, so neighbouring texels differ."""
    rng = np.random.default_rng(12000 + seed)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float64)
    img = np.stack([128 + 100 * np.sin(xx / (5.0 + c) + yy / (7.0 + 2 * c) + rng.uniform(0, 6)) for c in range(channels)], -1)
    img += rng.normal(0, 12, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)
