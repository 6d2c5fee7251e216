"""Float64 oracle of the 3DMM reconstruction (reference model_building.py:106-139 and the crop -> image affine of
utils/inference.py:127-138), with a per-element error scale, mirrors of the work plans of the two tensor-core
reconstruction kernels and the seeded parameters its tests feed them.  TEST INFRASTRUCTURE.

The contract is that of ``block64.py`` / ``gemm64.py``: ``reconstruct`` returns ``(want, S)`` and an output passes when
|got - want| <= tau * S at every element (``check64.worst``).

The tensor-core scheme (csrc/kernels_dense.cuh, ``syn_commit`` / ``pack_recon_tc`` in synergy_b200.cu).  Coefficient
k is multiplied by ascale_k = 2^(10 - e_k), where 2^e_k bounds |mean_k| + 8 |std_k| (2^10 when that bound is 0), and
face b is divided by its face scale fs_b, a power of two that is 1 unless the face's largest |alpha_k ascale_k| exceeds
60000 (then that value lands in [2^14, 2^15)).  Basis column k is divided by ascale_k and every (vertex, coordinate) row
c is multiplied by its row scale rs_c, which brings the row's max into [256, 512).  Both operands are split into fp16
hi + lo; the products hi*hi, hi*lo and lo*hi are accumulated in fp32 and the epilogue multiplies by fs_b / rs_c.

A split pair holds x to 2^-22 |x| while lo is a normal fp16 number; below that, lo (and for the smallest values hi)
falls into fp16's subnormals, whose spacing 2^-24 is absolute in scaled units.  The two bounds meet at a scaled
magnitude of 2^-24 / 2^-22 = 2^-2 (the floor of gemm64.py), so a coefficient is held to 2^-22 (|alpha_k| + eps_a[b, k])
and a basis entry to 2^-22 (|W_ck| + eps_W[c, k]), in the units of the model:

    eps_a[b, k] = 2^-2 fs_b / ascale_k    (at most 2^-11 of the 8-sigma bound, times the face scale)
    eps_W[c, k] = 2^-2 ascale_k / rs_c    (at most 2^-10 of the row's max |W_ck / ascale_k|, times ascale_k)

The omitted lo*lo pass is below 2^-22 |W_ck alpha_k|.  Every product enters S as (|W_ck| + eps_W)(|alpha_k| + eps_a), so
the absolute floors are charged at the same rate tau as the relative error of the pairs:

    S_c = |u_c| + sum_k (|W_ck| + eps_W[c, k]) (A_k + eps_a[b, k])
    S_i = sum_c |P_ic| S_c + |t_i|                                      (i = x, y, z of the posed vertex)

The de-whitening v * std + mean is rounded in fp32 and the rounding is relative to |v * std| + |mean|, not to the
(possibly cancelled) result, so with whitening A_k = |v_k std_k| + |mean_k|, and the pose entries P and t enter S with
the same magnitudes.  The y flip 121 - vy adds 121 + |vy| to S_y; the affine x * k + s maps S to |k| S + |s|.

The fp32 engine (``reconstruct_kernel``) is held to the same S with its own tau.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np

from oracle.check64 import worst  # noqa: F401  (the check the reconstruction tests apply)

IMG = 120
N_ALPHA = 50
CLAMP = 60000.0                         # split2_f16 (csrc/tc_common.cuh)
FLOOR = 2.0 ** -2                       # scaled magnitude below which the split's error is absolute
FACES = 64                              # kDnFaces: faces per tile
VTILE = 128                             # vertices per tile
RING = 4                                # kDnBSlots: alpha / pose ring of dense_recon_tc_kernel


def _exp(m: np.ndarray) -> np.ndarray:
    """e with m = f 2^e, f in [0.5, 1) (frexp) for fp32 magnitudes; 0 where m is 0 or not finite."""
    m = np.asarray(m, np.float32)
    _, e = np.frexp(m)
    return np.where((m > 0) & np.isfinite(m), e, 0).astype(np.int64)


def ascale(mean: np.ndarray, std: np.ndarray) -> np.ndarray:
    """ascale_k of syn_commit: 2^(10 - e_k), 2^e_k > |mean_k| + 8 |std_k| (fp32), (50,) float64."""
    m, s = np.asarray(mean, np.float32)[12:62], np.asarray(std, np.float32)[12:62]
    bound = np.abs(m) + np.float32(8) * np.abs(s)
    return np.exp2(10.0 - _exp(bound))


def row_scales(w: np.ndarray, asc: np.ndarray) -> np.ndarray:
    """rs_c of pack_recon_tc for basis rows w (R, 50) fp32: 2^(9 - e), 2^e > max_k |w_ck / ascale_k|; 1 for zero rows."""
    m = np.abs(np.asarray(w, np.float32) / asc.astype(np.float32)).max(axis=1)
    return np.where(m > 0, np.exp2(9.0 - _exp(m)), 1.0)


def dewhiten(params: np.ndarray, mean: np.ndarray, std: np.ndarray, whitening: bool) -> Tuple[np.ndarray, np.ndarray]:
    """(p, magnitude): the de-whitened parameters in float64 and the magnitude their fp32 rounding is relative to."""
    v = np.asarray(params, np.float32).astype(np.float64)
    if not whitening:
        return v, np.abs(v)
    vs = v * np.asarray(std, np.float32)[:62].astype(np.float64)
    mu = np.asarray(mean, np.float32)[:62].astype(np.float64)
    return vs + mu, np.abs(vs) + np.abs(mu)


def alpha_fp32(params: np.ndarray, mean: np.ndarray, std: np.ndarray, whitening: bool) -> np.ndarray:
    """The de-whitened fp32 coefficients dense_alpha_kernel computes (one rounding of v * std + mean), (B, 50)."""
    p, _ = dewhiten(params, mean, std, whitening)
    return p[:, 12:62].astype(np.float32)


def face_scales(params: np.ndarray, mean: np.ndarray, std: np.ndarray, whitening: bool) -> np.ndarray:
    """fs_b of dense_alpha_kernel, (B,) float64."""
    a = alpha_fp32(params, mean, std, whitening) * ascale(mean, std).astype(np.float32)
    m = np.abs(a).max(axis=1)
    big = (m > CLAMP) & np.isfinite(m)
    return np.where(big, np.exp2(_exp(m) - 15.0), 1.0)


def basis_rows(pack: Dict[str, np.ndarray], dense: bool) -> Tuple[np.ndarray, np.ndarray]:
    """(u (3N,), W (3N, 50)) fp32, rows interleaved x, y, z per vertex."""
    if dense:
        u, ws, we = pack['u'], pack['w_shp'], pack['w_exp']
    else:
        u, ws, we = pack['u_base'], pack['w_shp_base'], pack['w_exp_base']
    return np.asarray(u, np.float32).reshape(-1), np.concatenate([ws, we], 1).astype(np.float32)


def reconstruct(params: np.ndarray, pack: Dict[str, np.ndarray], dense: bool = False, whitening: bool = True,
                transform: bool = True, roi5: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """(want, S), both (B, 3, N) float64, of reconstruct_vertex_62 (``roi5`` (B, 5) = kx, sx, ky, sy, kz: the image-space
    variant, which always de-whitens and flips y)."""
    mean, std = pack['param_mean'], pack['param_std']
    u, w = basis_rows(pack, dense)
    asc = ascale(mean, std)
    p, pm = dewhiten(params, mean, std, whitening)
    fs = face_scales(params, mean, std, whitening)
    eps_a = FLOOR * fs[:, None] / asc[None, :]                                   # (B, 50)
    wabs = np.abs(w).astype(np.float64)
    wabs += FLOOR * asc[None, :] / row_scales(w, asc)[:, None]                   # |W| + eps_W, (3N, 50)
    alpha, amag = p[:, 12:62], pm[:, 12:62]
    shape = u.astype(np.float64)[None, :] + alpha @ w.astype(np.float64).T     # (B, 3N)
    s_shape = np.abs(u).astype(np.float64)[None, :] + (amag + eps_a) @ wabs.T
    b, n = shape.shape[0], shape.shape[1] // 3
    shape, s_shape = shape.reshape(b, n, 3), s_shape.reshape(b, n, 3)
    P, T = p[:, :12].reshape(b, 3, 4), pm[:, :12].reshape(b, 3, 4)
    want = np.einsum('bic,bnc->bin', P[:, :, :3], shape) + P[:, :, 3:]
    s = np.einsum('bic,bnc->bin', T[:, :, :3], s_shape) + T[:, :, 3:]
    if transform or roi5 is not None:
        s[:, 1] += IMG + 1 + np.abs(want[:, 1])
        want[:, 1] = IMG + 1 - want[:, 1]
    if roi5 is not None:
        r = np.asarray(roi5, np.float32).astype(np.float64)
        k, off = r[:, [0, 2, 4]][:, :, None], np.concatenate([r[:, [1, 3]], np.zeros((b, 1))], 1)[:, :, None]
        want = want * k + off
        s = s * np.abs(k) + np.abs(off)
    return want, s


def reconstruct_chunked(params, pack, chunk: int = 64, **kw) -> Tuple[np.ndarray, np.ndarray]:
    """``reconstruct`` in chunks of ``chunk`` faces (the dense basis is 53 215 x 3 rows)."""
    parts = [reconstruct(params[i:i + chunk], pack, roi5=None if kw.get('roi5') is None else kw['roi5'][i:i + chunk],
                         **{k: v for k, v in kw.items() if k != 'roi5'}) for i in range(0, len(params), chunk)]
    return np.concatenate([q[0] for q in parts]), np.concatenate([q[1] for q in parts])


# ---- inputs -----------------------------------------------------------------------------------------------------------

RESNET_SCALED = 23010.0                   # |alpha * ascale| the random ResNet-50 checkpoint reaches


def random_params(b, seed, spread=1.0):
    """Whitened parameters: distinct faces within a few sigma."""
    return (np.random.default_rng(seed).standard_normal((b, 62)) * spread).astype(np.float32)


def roi_rows(b, seed):
    rng = np.random.default_rng(seed)
    k = rng.uniform(0.3, 4.0, (b, 3))
    s = rng.uniform(-50.0, 800.0, (b, 2))
    return np.stack([k[:, 0], s[:, 0], k[:, 1], s[:, 1], k[:, 2]], 1).astype(np.float32)


def _whiten(p_raw, pack):
    mean, std = pack['param_mean'][:62].astype(np.float64), pack['param_std'][:62].astype(np.float64)
    return ((p_raw - mean) / np.where(std == 0, 1.0, std)).astype(np.float32)


def magnitude_params(pack, beyond):
    """(params, whitening) with coefficients at the magnitudes the alpha scale has to cover.  ``beyond`` = False: the
    mean, +-8 sigma, the ResNet-50 magnitude, just below the fp16 clamp 60000 / ascale_k, and translations that put the
    vertices around y = 121 (the flip cancels).  ``beyond`` = True: just above the clamp, one coefficient far above it
    next to tiny ones, and raw coefficients (whitening off) far beyond it, including the coefficient of the stress
    model whose mean and std are 0."""
    from oracle.synth_model import STRESS_ZERO_COEF
    mean, std = pack['param_mean'][:62].astype(np.float64), pack['param_std'][:62].astype(np.float64)
    lim = CLAMP / ascale(mean, std)                                     # |alpha_k| at the clamp
    sign = np.where(np.arange(50) % 2, -1.0, 1.0)
    base = random_params(8, 91, 0.5).astype(np.float64)
    rows = []

    def face(alpha, i):
        p = base[i % 8].copy() * std + mean
        p[12:62] = alpha
        return p

    if not beyond:
        rows += [face(mean[12:62], 0), face(mean[12:62] + 8 * std[12:62], 1), face(mean[12:62] - 8 * std[12:62], 2)]
        rows += [face(sign * RESNET_SCALED / ascale(mean, std), 3), face(0.999 * sign * lim, 4),
                 face(-0.999 * sign * lim, 5)]
        for i in range(4):
            p = face(mean[12:62] + 2 * std[12:62] * np.random.default_rng(i).standard_normal(50), 6 + i)
            p[7] = 121.0 + 8.0 * i                                      # t_y: vy = 121 within the face
            rows.append(p)
        return _whiten(np.stack(rows), pack), True
    rows += [face(1.001 * sign * lim, 0), face(-1.5 * sign * lim, 1)]
    p = face(mean[12:62] + 1e-3 * std[12:62], 2)
    p[12] = 4.0 * lim[0]                                                # huge next to tiny
    rows.append(p)
    p = face(mean[12:62] + 1e-6 * std[12:62], 3)
    p[12 + 40] = -1e3 * lim[40]
    rows.append(p)
    rows += [face(3.0 * sign * lim, 4), face(-40.0 * lim, 5)]
    for i, a in enumerate((100.0, -1000.0, 58.0, 1e5)):
        p = face(mean[12:62], 6 + i)
        p[12 + STRESS_ZERO_COEF] = a                                    # ascale 2^10 when mean = std = 0
        rows.append(p)
    return np.stack(rows).astype(np.float32), False


# ---- work plans -----------------------------------------------------------------------------------------------------

def dense_plan(batch: int, sms: int, n_vert: int) -> Dict[str, int]:
    """dense_recon_fm_kernel (run_reconstruct_tc in synergy_b200.cu; the band split at the top of the kernel): face tiles,
    vertex bands per face tile, vertex tiles per band, grid, CTAs with no items, items of the last non-empty band."""
    ftiles, vtiles = -(-batch // FACES), -(-n_vert // VTILE)
    grid = ftiles * min(max(1, sms // ftiles), vtiles)
    bands = max(1, grid // ftiles)
    band_len = -(-vtiles // bands)
    used = -(-vtiles // band_len)
    return dict(ftiles=ftiles, vtiles=vtiles, bands=bands, band_len=band_len, grid=grid, idle=(bands - used) * ftiles,
                last_band=vtiles - (used - 1) * band_len)


def sparse_plan(batch: int, sms: int, n_pts: int) -> Dict[str, int]:
    """dense_recon_tc_kernel: items (vertex tile, face tile), vertex-tile major, split into contiguous runs of ``per``
    items over min(items, SMs) CTAs; ``crossings`` is the largest number of vertex-tile changes inside one CTA's run."""
    ftiles, vtiles = -(-batch // FACES), -(-n_pts // VTILE)
    items = ftiles * vtiles
    grid = min(items, sms)
    per = -(-items // grid)
    cross = 0
    for c in range(grid):
        i0, i1 = min(c * per, items), min(c * per + per, items)
        if i1 > i0:
            cross = max(cross, (i1 - 1) // ftiles - i0 // ftiles)
    return dict(ftiles=ftiles, vtiles=vtiles, grid=grid, per=per, crossings=cross)


def choose_dense_cases(sms: int, nver: int = 53215) -> Dict[str, Tuple[int, int]]:
    """(batch, n_vert) per dense plan kind; the narrow bases keep the output under 200 MB."""
    return {'small_idle': (37, nver),                   # one face tile, more bands than needed: idle CTAs
            'ragged_multi': (4 * FACES + 9, nver),      # ragged last face tile, bands of several items
            'short_last': (3 * FACES, nver),
            'one_item': (5 * FACES - 3, 8 * VTILE - 5),
            'one_band': ((sms // 2 + 1) * FACES - 17, 1000),
            'grid_gt_sms': (sms * FACES + 1, 129)}


def check_dense_case(kind: str, batch: int, n_vert: int, sms: int) -> None:
    """Assert that (batch, n_vert) produces the plan ``kind`` names."""
    p = dense_plan(batch, sms, n_vert)
    if kind == 'small_idle':
        assert batch <= FACES and p['idle'] > 0, p
    elif kind == 'ragged_multi':
        assert batch % FACES and p['band_len'] >= 2, p
    elif kind == 'short_last':
        assert p['band_len'] >= 2 and 0 < p['last_band'] < p['band_len'], p
    elif kind == 'one_item':
        assert p['band_len'] == 1 and p['bands'] == p['vtiles'] and batch % FACES, p
    elif kind == 'one_band':
        assert p['bands'] == 1 and p['grid'] == p['ftiles'] <= sms and batch % FACES, p
    elif kind == 'grid_gt_sms':
        assert p['grid'] > sms and p['bands'] == 1, p
    else:
        raise ValueError(kind)


def choose_sparse_cases(sms: int) -> Dict[str, Tuple[int, int]]:
    """(batch, n_pts) per sparse plan kind: the B ring wraps past its second lap (more than 2 * RING items per CTA);
    a CTA's run crosses a vertex-tile boundary; every item of a run is a new vertex tile (the meta double buffer)."""
    return {'ring_wrap': (2 * RING * FACES * sms + 3 * FACES + 5, 68),
            'tile_cross': (FACES * (sms // 2 | 1), 300),
            'meta_cycle': (FACES, (3 * sms + 7) * VTILE - 11)}


def check_sparse_case(kind: str, batch: int, n_pts: int, sms: int) -> None:
    p = sparse_plan(batch, sms, n_pts)
    if kind == 'ring_wrap':
        assert p['per'] > 2 * RING and p['grid'] == sms, p
    elif kind == 'tile_cross':
        assert p['vtiles'] > 1 and p['crossings'] >= 1 and n_pts == 300, p
    elif kind == 'meta_cycle':
        assert p['crossings'] >= 2 and p['ftiles'] == 1, p
    else:
        raise ValueError(kind)
