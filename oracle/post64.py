"""Float64 restatements of the kernels at the two ends of the path: pose decode, FaceBoxes box decode and the two
training losses.  TEST INFRASTRUCTURE.

Each function returns ``(want, S)``: the value in float64 and its first-order error scale, the sum of the absolute
values of the terms entering every rounded step of the kernel's sequence (``check64`` convention), so that every
element is held to |got - want| <= TAU * S.  The NMS kernels return index lists; their oracles are the numpy and C
restatements of ``render_port``.

Pose decode (``pose_decode_kernel``) has two checks:
  * ``pose_angles_seq``: the double-precision angles of the fp32 rotation the kernel claims to compute
    (``pose_rotation_f32``: whitening, three-term sums in order, sqrt, divisions, cross product, elementwise float32
    numpy, no BLAS and no fused multiply-add).  S is a few double ulps times the condition of asin / atan2, so one fp32
    slip anywhere in the kernel's R measures >= 1e6 TAU.
  * ``pose_angles_acc``: the angles of R computed in float64 from the same fp32 P.  S carries the fp32 rounding of R
    through the normalisation, the cross product and the condition of asin / atan2 -- the pose is as accurate as its
    fp32 input allows.
Both take the branch the kernel takes, decided by the fp32 bits of R20: |R20| >= 1 is the gimbal-lock branch with
R20's sign (the reference's own value at +-1, where it is defined; ``math.asin`` raises beyond).
"""
from __future__ import annotations

from typing import Tuple

import numpy as np

from oracle.check64 import f32_dot3

F32 = np.float32
U32 = 2.0 ** -24                 # fp32 unit round-off; the accuracy S of an angle is floored with it near the lock
DEG = 180.0 / np.pi
Pair = Tuple[np.ndarray, np.ndarray]


# ---- pose decode -------------------------------------------------------------------------------------------------------
def pose_p(params: np.ndarray, mean: np.ndarray, std: np.ndarray) -> np.ndarray:
    """P = (param * std + mean)[:12] in fp32, one rounding per operation: (B, 12) float32."""
    p = np.asarray(params, F32)[:, :12]
    return (p * np.asarray(std, F32)[:12]) + np.asarray(mean, F32)[:12]


def _norm_f32(v: np.ndarray) -> np.ndarray:
    return np.sqrt(f32_dot3(v, v))


def pose_rotation_f32(P: np.ndarray) -> np.ndarray:
    """The kernel's fp32 R (B,3,3): rows r1 = P[0:3] / |P[0:3]|, r2 = P[4:7] / |P[4:7]|, r3 = np.cross(r1, r2)."""
    P = np.asarray(P, F32)
    with np.errstate(all='ignore'):
        r1 = P[:, 0:3] / _norm_f32(P[:, 0:3])[:, None]
        r2 = P[:, 4:7] / _norm_f32(P[:, 4:7])[:, None]
        r3 = np.stack([r1[:, 1] * r2[:, 2] - r1[:, 2] * r2[:, 1],
                       r1[:, 2] * r2[:, 0] - r1[:, 0] * r2[:, 2],
                       r1[:, 0] * r2[:, 1] - r1[:, 1] * r2[:, 0]], 1)
    return np.stack([r1, r2, r3], 1)


def _lock(r20_f32: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(R20 >= 1, R20 <= -1) on the fp32 bits: the two gimbal-lock branches (NaN takes neither)."""
    r = np.asarray(r20_f32, F32)
    return r >= 1, r <= -1


def pose_angles_seq(R32: np.ndarray) -> Pair:
    """matrix2angle_corr in double on the fp32 R, as the kernel evaluates it: (B,3) degrees and S (double ulps times
    the condition of each step; atan2 of two quotients by the same cos(x) does not depend on cos(x)'s rounding)."""
    R = np.asarray(R32, F32).astype(np.float64)
    hi, lo = _lock(R32[:, 2, 0])
    with np.errstate(all='ignore'):
        x = np.arcsin(R[:, 2, 0])
        c = np.cos(x)
        y = np.arctan2(R[:, 1, 2] / c, R[:, 2, 2] / c)
        z = np.arctan2(R[:, 0, 1] / c, R[:, 0, 0] / c)
    x = np.where(hi, -np.pi / 2, np.where(lo, np.pi / 2, x))
    y = np.where(hi, np.arctan2(-R[:, 0, 1], -R[:, 0, 2]), np.where(lo, np.arctan2(R[:, 0, 1], R[:, 0, 2]), y))
    z = np.where(hi | lo, 0.0, z)
    ang = np.stack([x, y, z], 1)
    want = ang * 180 / np.pi
    # asin on an exact input: |x|; atan2 of arguments with one relative rounding each: |y| + 1 (radians); then the two
    # roundings of * 180 / pi
    s = np.stack([np.abs(x), np.abs(y) + 1, np.abs(z) + 1], 1)
    return want, (s + 2 * np.abs(ang)) * DEG


def pose_rotation_s(P: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """R in float64 from the fp32 P (B,3,3) and the S of the kernel's fp32 R against it."""
    P = np.asarray(P, F32).astype(np.float64)

    def row(v):
        sq = v * v
        n2 = sq.sum(1)
        n = np.sqrt(n2)
        s_n2 = 2 * n2 + sq[:, 0] + sq[:, 1]                  # three squares, then (a^2 + b^2) and + c^2
        s_n = s_n2 / (2 * n) + n
        r = v / n[:, None]
        return r, np.abs(r) * (s_n / n)[:, None] + np.abs(r)
    with np.errstate(all='ignore'):
        (a, sa), (b, sb) = row(P[:, 0:3]), row(P[:, 4:7])
        r3, s3 = [], []
        for i, j in ((1, 2), (2, 0), (0, 1)):
            t1, t2 = a[:, i] * b[:, j], a[:, j] * b[:, i]
            r3.append(t1 - t2)
            s3.append(np.abs(b[:, j]) * sa[:, i] + np.abs(a[:, i]) * sb[:, j] + np.abs(b[:, i]) * sa[:, j]
                      + np.abs(a[:, j]) * sb[:, i] + 2 * (np.abs(t1) + np.abs(t2)))
    return np.stack([a, b, np.stack(r3, 1)], 1), np.stack([sa, sb, np.stack(s3, 1)], 1)


def _atan2_s(a, b, sa, sb):
    """First-order S of atan2(a, b) for S(a), S(b); unbounded (inf) where a = b = 0."""
    den = a * a + b * b
    with np.errstate(all='ignore'):
        return np.where(den > 0, (np.abs(b) * sa + np.abs(a) * sb) / den, np.inf)


def pose_angles_acc(P: np.ndarray) -> Pair:
    """The angles of the float64 R of the fp32 P, on the branch the fp32 R20 selects: (B,3) degrees and S, the fp32
    rounding of R carried through asin / atan2 (S_x = S_R20 / sqrt(1 - R20^2), floored near the lock where asin's
    derivative is unbounded), plus a double-rounding term."""
    R, S = pose_rotation_s(P)
    hi, lo = _lock(pose_rotation_f32(P)[:, 2, 0])
    r20 = np.clip(R[:, 2, 0], -1, 1)
    x = np.arcsin(r20)
    y = np.arctan2(R[:, 1, 2], R[:, 2, 2])                 # cos(x) > 0 divides both
    z = np.arctan2(R[:, 0, 1], R[:, 0, 0])
    sx = S[:, 2, 0] / np.sqrt(np.maximum(1 - r20 * r20, U32 * S[:, 2, 0]))
    sy = _atan2_s(R[:, 1, 2], R[:, 2, 2], S[:, 1, 2], S[:, 2, 2])
    sz = _atan2_s(R[:, 0, 1], R[:, 0, 0], S[:, 0, 1], S[:, 0, 0])
    s_lock = _atan2_s(R[:, 0, 1], R[:, 0, 2], S[:, 0, 1], S[:, 0, 2])
    lock = hi | lo
    x = np.where(hi, -np.pi / 2, np.where(lo, np.pi / 2, x))
    y = np.where(hi, np.arctan2(-R[:, 0, 1], -R[:, 0, 2]), np.where(lo, np.arctan2(R[:, 0, 1], R[:, 0, 2]), y))
    z = np.where(lock, 0.0, z)
    sx, sy, sz = np.where(lock, 0.0, sx), np.where(lock, s_lock, sy), np.where(lock, 0.0, sz)
    ang = np.stack([x, y, z], 1)
    return ang * DEG, (np.stack([sx, sy, sz], 1) + 2.0 ** -29 * (np.abs(ang) + 1)) * DEG


def pose_t3d(P: np.ndarray, roi5: np.ndarray = None) -> Pair:
    """t3d = P[:, 3] (B,3), moved to image coordinates with the fp32 roi rows: t * k + s, two fp32 roundings."""
    P = np.asarray(P, F32).astype(np.float64)
    t = P[:, [3, 7, 11]].copy()
    s = np.zeros_like(t)
    if roi5 is not None:
        r = np.asarray(roi5, F32).astype(np.float64)
        for c, (k, o) in enumerate(((0, 1), (2, 3))):
            m = t[:, c] * r[:, k]
            t[:, c] = m + r[:, o]
            s[:, c] = 2 * np.abs(m) + np.abs(r[:, o])
    return t, s


# ---- FaceBoxes box decode --------------------------------------------------------------------------------------------------
def priors(h: int, w: int) -> np.ndarray:
    """prior_box.py:23-43 in Python doubles rounded to fp32 once, (P,4) [cx cy s_kx s_ky]."""
    out = []
    for step, sizes in ((32, (32, 64, 128)), (64, (256,)), (128, (512,))):
        for i in range(-(-h // step)):
            for j in range(-(-w // step)):
                for ms in sizes:
                    offs = {32: (0, 0.25, 0.5, 0.75), 64: (0, 0.5)}.get(ms, (0.5,))
                    out += [((j + ox) * step / w, (i + oy) * step / h, ms / w, ms / h) for oy in offs for ox in offs]
    return np.asarray(out, np.float64).astype(F32)


def decode_order(conf: np.ndarray, thresh: float, top_k: int) -> np.ndarray:
    """Prior indices of the rows of the kernel's output: scores > thresh in descending order, ties by the higher index
    first (a stable ascending argsort read backwards), the first top_k."""
    s = np.asarray(conf, F32)[:, 1]
    idx = np.nonzero(s > F32(thresh))[0]
    order = idx[np.argsort(s[idx], kind='stable')][::-1]
    return order[:top_k]


def decode_f32(loc: np.ndarray, pri: np.ndarray, bsw: float, bsh: float, scale: float) -> np.ndarray:
    """box_utils.py:191-194 + FaceBoxes.py:104 in fp32 numpy, one rounding per operation: (n,4).  Used for the classes
    of non-finite outputs, which follow fp32 overflow."""
    l, p = np.asarray(loc, F32), np.asarray(pri, F32)
    with np.errstate(all='ignore'):
        cx = p[:, 0] + l[:, 0] * F32(0.1) * p[:, 2]
        cy = p[:, 1] + l[:, 1] * F32(0.1) * p[:, 3]
        bw, bh = p[:, 2] * np.exp(l[:, 2] * F32(0.2)), p[:, 3] * np.exp(l[:, 3] * F32(0.2))
        x1, y1 = cx - bw / F32(2), cy - bh / F32(2)
        x2, y2 = bw + x1, bh + y1
        return np.stack([x1 * F32(bsw) / F32(scale), y1 * F32(bsh) / F32(scale),
                         x2 * F32(bsw) / F32(scale), y2 * F32(bsh) / F32(scale)], 1)


def decode(loc: np.ndarray, pri: np.ndarray, bsw: float, bsh: float, scale: float) -> Pair:
    """The same in float64 on the fp32 inputs and constants (0.1f, 0.2f): (n,4) and S.  exp's S is e * (1 + |0.2 l|):
    its own rounding and that of its argument."""
    l, p = np.asarray(loc, F32).astype(np.float64), np.asarray(pri, F32).astype(np.float64)
    v1, v2 = float(F32(0.1)), float(F32(0.2))
    bsw, bsh, scale = float(F32(bsw)), float(F32(bsh)), float(F32(scale))
    with np.errstate(all='ignore'):
        out, s = [], []
        for c, k in ((0, 0), (1, 1)):                    # centre: p + (l * 0.1) * s_k, three roundings
            m = l[:, c] * v1 * p[:, 2 + k]
            out.append(p[:, k] + m)
            s.append(np.abs(p[:, k]) + 3 * np.abs(m))
        for c, k in ((2, 0), (3, 1)):                    # size: s_k * exp(l * 0.2)
            a = l[:, c] * v2
            e = np.exp(a)
            out.append(p[:, 2 + k] * e)
            s.append(np.abs(out[-1]) * (2 + np.abs(a)))
        cx, cy, bw, bh = out
        scx, scy, sbw, sbh = s
        x1, y1 = cx - bw / 2, cy - bh / 2
        sx1, sy1 = scx + sbw / 2 + np.abs(cx) + np.abs(bw / 2), scy + sbh / 2 + np.abs(cy) + np.abs(bh / 2)
        x2, y2 = bw + x1, bh + y1
        sx2, sy2 = sbw + sx1 + np.abs(bw) + np.abs(x1), sbh + sy1 + np.abs(bh) + np.abs(y1)
        want, sw = [], []
        for v, sv, b in ((x1, sx1, bsw), (y1, sy1, bsh), (x2, sx2, bsw), (y2, sy2, bsh)):
            want.append(v * b / scale)
            sw.append((sv + 2 * np.abs(v)) * b / scale)  # the scale multiply and divide
    return np.stack(want, 1), np.stack(sw, 1)


# ---- training losses ---------------------------------------------------------------------------------------------------
def wing_loss(pred: np.ndarray, target: np.ndarray, omega: float = 10.0, epsilon: float = 2.0) -> Pair:
    """WingLoss (loss_definition.py:15-27): the mean of omega * log(1 + d / eps) (d < omega) and d - C (d >= omega) over
    the deltas that pass one of the comparisons (a NaN delta passes neither), C = omega - omega * log(1 + omega / eps)
    in double rounded to fp32.  S = sum of |terms| / n, each term's own rounding and that of d = |t - p| carried by its
    slope."""
    p, t = np.asarray(pred, F32).reshape(-1), np.asarray(target, F32).reshape(-1)
    with np.errstate(all='ignore'):
        d32 = np.abs(t - p)
        lin, log_ = d32 >= F32(omega), d32 < F32(omega)
        d = np.abs(t.astype(np.float64) - p.astype(np.float64))
        C = float(F32(omega - omega * np.log(1 + omega / epsilon)))
        terms = np.where(log_, omega * np.log1p(d / epsilon), d - C)
        s_d = np.abs(t.astype(np.float64)) + np.abs(p.astype(np.float64))       # the subtraction giving d
        # log branch: d / eps, 1 + q (relative rounding -> omega absolute), log and * omega; linear branch: d - C
        s = np.where(log_, omega / (epsilon + d) * s_d + omega + 2 * np.abs(terms), s_d + d + abs(C))
        keep = lin | log_
        n = int(keep.sum())
        if n == 0:
            return np.asarray(np.nan), np.asarray(0.0)
        want = terms[keep].sum() / n
        return np.asarray(want), np.asarray(s[keep].sum() / n + abs(want))


def param_loss(inp: np.ndarray, tg: np.ndarray, mode: int = 0) -> Pair:
    """ParamLoss (loss_definition.py:35-42) per sample, with the kernel's sequential fp32 sums: (B,) and S."""
    x, t = np.asarray(inp, np.float64), np.asarray(tg, np.float64)
    if mode == 0:
        parts = ((x[:, :12], t[:, :12], 12.0), (x[:, 12:62], t[:, 12:62], 50.0))
    else:
        parts = ((x[:, :50], t[:, 12:62], 50.0),)
    m = np.zeros(x.shape[0])
    sm = np.zeros(x.shape[0])
    for xs, ts, cnt in parts:
        d = xs - ts
        sq = d * d
        run = np.cumsum(sq, 1)
        # each delta's rounding carried by the square (2 |d| (|x| + |t|)), the square's own, every partial sum, the divide
        s_sum = (2 * np.abs(d) * (np.abs(xs) + np.abs(ts)) + sq).sum(1) + run[:, 1:].sum(1)
        m += run[:, -1] / cnt
        sm += (s_sum + run[:, -1]) / cnt
    if len(parts) == 2:
        sm += m                                          # the add of the two means
    want = np.sqrt(m)
    with np.errstate(all='ignore'):
        s = np.where(m > 0, sm / (2 * want), 0.0) + want
    return want, s


# ---- pose cases --------------------------------------------------------------------------------------------------------
def _whiten(P: np.ndarray, mean: np.ndarray, std: np.ndarray) -> np.ndarray:
    """(B,62) float32 params whose first 12 whiten the (B,12) camera rows ``P`` (the rest zero)."""
    out = np.zeros((P.shape[0], 62), F32)
    out[:, :12] = ((np.asarray(P, np.float64) - np.asarray(mean, np.float64)[:12]) / np.asarray(std, np.float64)[:12])
    return out


def _camera(r1: np.ndarray, r2: np.ndarray, rng) -> np.ndarray:
    P = np.zeros((r1.shape[0], 12))
    P[:, 0:3], P[:, 4:7], P[:, 8:11] = r1, r2, np.cross(r1, r2)
    P[:, [3, 7, 11]] = rng.uniform(-200, 200, (r1.shape[0], 3))
    return P


def pose_cases_so3(mean, std, n: int, seed: int = 0) -> np.ndarray:
    """``n`` params whose camera rows are those of rotations drawn uniformly on SO(3) (unit quaternions), each row scaled
    by its own 10^U(-4, 2) and, for every other face, the second row sheared by up to half the first."""
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((n, 4))
    w, x, y, z = (q / np.linalg.norm(q, axis=1, keepdims=True)).T
    r1 = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], 1)
    r2 = np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], 1)
    shear = np.where(np.arange(n) % 2 == 1, rng.uniform(-0.5, 0.5, n), 0.0)
    r2 = r2 + shear[:, None] * r1
    s = 10.0 ** rng.uniform(-4, 2, (n, 2))
    return _whiten(_camera(r1 * s[:, :1], r2 * s[:, 1:], rng), mean, std)


def pose_cases_lock(mean, std, seed: int = 0, ulps: int = 64) -> Tuple[np.ndarray, np.ndarray]:
    """Yaw sweeps at +-90 degrees (camera rows with a first column near 0), searched on the host with the kernel's fp32
    sequence so that R20 takes every fp32 value within ``ulps`` ulps of +-1, exactly +-1, and every value above 1 in
    magnitude that the sweep reaches.  Returns (params (B,62), their fp32 R20)."""
    rng = np.random.default_rng(seed)
    picked = {}
    for _ in range(40):
        m = 50000
        th = rng.uniform(0, 2 * np.pi, m)
        eps = 10.0 ** rng.uniform(-6, -2.2, (m, 2)) * rng.choice([-1, 1], (m, 2))
        eps[rng.random(m) < 0.3] = 0.0
        r1 = np.stack([eps[:, 0], np.cos(th), np.sin(th)], 1)
        r2 = np.stack([eps[:, 1], -np.sin(th), np.cos(th)], 1) * rng.choice([-1, 1], (m, 1))
        s = 10.0 ** rng.uniform(-1, 1.5, (m, 2))
        p = _whiten(_camera(r1 * s[:, :1], r2 * s[:, 1:], rng), mean, std)
        r20 = pose_rotation_f32(pose_p(p, mean, std))[:, 2, 0]
        for v in np.unique(r20):
            if abs(float(v)) >= 1 - ulps * U32 and float(v) not in picked:
                picked[float(v)] = p[np.nonzero(r20 == v)[0][0]]
    keys = sorted(picked)
    return np.stack([picked[k] for k in keys]), np.asarray(keys, F32)


def pose_cases_special() -> np.ndarray:
    """Camera rows (B,12) for identity whitening (mean 0, std 1): zero rows, and rows whose squares overflow or
    underflow fp32 (to inf, to 0, to subnormals), alone and mixed with ordinary rows."""
    rows = [np.zeros(3), np.array([1e20, 0, 0]), np.array([3e19, -2e19, 1e19]), np.array([1e-23, 0, 0]),
            np.array([1e-23, -2e-23, 3e-24]), np.array([1e-20, 2e-20, 0]), np.array([3e-19, 1e-19, -2e-19]),
            np.array([0.6, 0.8, 0]), np.array([0, -0.28, 0.96]), np.array([np.inf, 1, 0]), np.array([3.4e38, 1, 0])]
    P = [np.concatenate([a, [5.0], b, [-7.0], [0, 0, 0, 1.5]]) for a in rows for b in rows]
    return np.asarray(P, np.float64).astype(F32)


# ---- NMS cases ---------------------------------------------------------------------------------------------------------
def nms_cases(n, seed):
    """Random boxes with NaN / +-inf coordinates (as a decode past expf's overflow gives them) and zero-overlap pairs."""
    rng = np.random.default_rng(seed)
    c, wh = rng.uniform(0, 150, (n, 2)), rng.uniform(5, 60, (n, 2))
    d = np.hstack([c - wh / 2, c + wh / 2, rng.permutation(n)[:, None] / n]).astype(np.float32)
    k = rng.choice(n, n // 5, replace=False)
    d[k[0::3], 0], d[k[0::3], 2] = -np.inf, np.nan                  # x1 = -inf, x2 = inf + -inf
    d[k[1::3], rng.integers(0, 4, len(k[1::3]))] = np.nan
    d[k[2::3], 2], d[k[2::3], 3] = np.inf, np.inf
    far = rng.choice(n, n // 10, replace=False)                      # boxes that touch nothing
    d[far, :4] = (np.arange(len(far))[:, None] * 1000 + 5000 + np.array([0, 0, 10, 10])).astype(np.float32)
    return d
