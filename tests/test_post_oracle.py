"""CPU checks of oracle/post64.py, the float64 restatements of the pose decode, box decode and loss kernels: agreement
with the reference restatement and the golden vectors on ordinary inputs, the branch and S claims, negative controls
that must fail the bars, and the NMS algorithm on non-finite boxes."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from oracle import post64, render_port
from oracle import reference_port as rp
from oracle.check64 import ratio
from oracle.stage_check import TAU

HERE = os.path.dirname(os.path.abspath(__file__))
T = TAU['post64']


@pytest.fixture(scope='module')
def whitening(synth_pack):
    return np.asarray(synth_pack.param_mean, np.float32)[:62], np.asarray(synth_pack.param_std, np.float32)[:62]


def _pose(params, mean, std):
    P = post64.pose_p(params, mean, std)
    return P, post64.pose_angles_seq(post64.pose_rotation_f32(P)), post64.pose_angles_acc(P)


def test_pose_oracle_agrees_with_reference_and_golden(whitening):
    mean, std = whitening
    prm = post64.pose_cases_so3(mean, std, 300, seed=3)
    P, (ws, ss), (wa, sa) = _pose(prm, mean, std)
    assert ratio(ws, wa, sa).max() <= T['pose']                    # the fp32 sequence is as accurate as its input allows
    pack = dict(param_mean=mean, param_std=std)
    ref = np.array([rp.predict_pose(prm[i], pack, [0, 0, 120, 120])[0] for i in range(len(prm))])
    assert ratio(ref, wa, sa).max() <= T['pose']                   # numpy's BLAS norm: same bar
    from golden.vectors import load_ref_vectors
    gold = load_ref_vectors()
    roi = [30.2, 41.7, 211.4, 222.9, 0.99]
    from synergynet_b200 import inference
    P, _, (wa, sa) = _pose(gold['params'][:1], mean, std)
    assert ratio(gold['np_pose_angles'][None], wa, sa).max() <= T['pose']
    t, st = post64.pose_t3d(P, inference.roi_affine([roi]))
    assert ratio(gold['np_pose_t3d'][None], t, st).max() <= T['t3d']


def test_pose_lock_sweep_branches(whitening):
    """The sweep reaches every fp32 R20 within 64 ulps of +-1, exactly +-1 and beyond; |R20| >= 1 takes the lock branch
    of R20's sign (x = -90 for +1, +90 for -1), the reference raises beyond 1 and gives that same value at +-1."""
    mean, std = whitening
    prm, r20 = post64.pose_cases_lock(mean, std)
    k = np.round((1 - np.abs(r20.astype(np.float64))) / post64.U32)
    for sign in (1, -1):
        assert set(range(0, 65)) <= set(k[np.sign(r20) == sign].tolist())
        assert (k[np.sign(r20) == sign] < 0).any()
    P, (ws, ss), (wa, sa) = _pose(prm, mean, std)
    assert np.isfinite(ws).all() and np.isfinite(ss).all() and np.isfinite(sa).all()
    assert ratio(ws, wa, sa).max() <= T['pose']
    lock = np.abs(r20) >= 1
    assert np.array_equal(ws[lock, 0], np.where(r20[lock] > 0, -90.0, 90.0)) and (ws[lock, 2] == 0).all()
    R = post64.pose_rotation_f32(P).astype(np.float64)
    for i in np.nonzero(lock)[0]:
        if abs(r20[i]) > 1:
            with pytest.raises(ValueError):
                rp.matrix2angle_corr(R[i])
        else:
            assert np.array_equal(rp.matrix2angle_corr(R[i]), ws[i])
    # away from the lock, S_x carries asin's condition: S grows as 1 / sqrt(1 - R20^2)
    near = (k >= 1) & (k <= 64)
    assert (sa[near, 0] > 100 * sa[~lock & ~near, 0].max()).all() if (~lock & ~near).any() else True


def test_pose_special_rows_follow_fp32():
    """Zero, overflowing and underflowing rows: NaN, inf and 0 where numpy's fp32 gives them."""
    P = post64.pose_cases_special()
    R = post64.pose_rotation_f32(P)
    ws, _ = post64.pose_angles_seq(R)
    assert np.isnan(ws).any() and np.isfinite(ws).any()
    assert np.isnan(ws[0]).all()                                   # zero rows: 0 / 0
    assert np.isnan(R[0]).all()
    assert (R[1 * 11 + 7, 0] == 0).all()                           # 1e20: the squares overflow, 1e20 / inf = 0
    assert np.isposinf(R[3 * 11 + 7, 0, 0])                        # 1e-23: the squares underflow to 0, 1e-23 / 0 = inf
    assert np.isfinite(R[5 * 11 + 7, 0]).all()                     # 1e-20: subnormal squares, no flush to zero


def test_negative_controls_fail_the_bar(whitening):
    mean, std = whitening
    prm = post64.pose_cases_so3(mean, std, 300, seed=4)
    P, (ws, ss), (wa, sa) = _pose(prm, mean, std)
    # the deleted host helper: float32 trigonometry on the fp32 R
    R = post64.pose_rotation_f32(P)
    x = np.arcsin(R[:, 2, 0])
    c = np.cos(x)
    f32 = np.stack([x, np.arctan2(R[:, 1, 2] / c, R[:, 2, 2] / c), np.arctan2(R[:, 0, 1] / c, R[:, 0, 0] / c)], 1)
    assert f32.dtype == np.float32
    assert ratio(f32 * np.float32(180 / np.pi), wa, sa).max() > 10 * T['pose']
    # an FMA-contracted norm: fma(c, c, fma(b, b, a * a)) -- exact products in double, one rounding per FMA
    def fma_norm(v):
        v = v.astype(np.float64)
        s = (v[:, 0] * v[:, 0]).astype(np.float32).astype(np.float64)
        s = (s + v[:, 1] * v[:, 1]).astype(np.float32).astype(np.float64)
        return np.sqrt((s + v[:, 2] * v[:, 2]).astype(np.float32))
    r1, r2 = P[:, 0:3] / fma_norm(P[:, 0:3])[:, None], P[:, 4:7] / fma_norm(P[:, 4:7])[:, None]
    Rf = np.stack([r1, r2, np.cross(r1, r2)], 1)
    assert Rf.dtype == np.float32
    wf, _ = post64.pose_angles_seq(Rf)
    assert ratio(wf, ws, ss).max() > 1e6 * T['pose_seq']
    # a decode whose exp is 64 ulps off
    rng = np.random.default_rng(0)
    pri = post64.priors(100, 150)
    loc = rng.standard_normal((pri.shape[0], 4)).astype(np.float32) * 3
    want, s = post64.decode(loc, pri, 150, 100, 1.0)
    got = post64.decode_f32(loc, pri, 150, 100, 1.0)
    assert ratio(got, want, s).max() <= T['decode']
    bad_exp = lambda a: np.exp(a) * np.float32(1 + 64 * 2.0 ** -23)
    l = loc.astype(np.float32)
    bw = pri[:, 2] * bad_exp(l[:, 2] * np.float32(0.2))
    cx = pri[:, 0] + l[:, 0] * np.float32(0.1) * pri[:, 2]
    x1 = cx - bw / np.float32(2)
    assert ratio((bw + x1) * np.float32(150), want[:, 2], s[:, 2]).max() > T['decode']


def test_decode_oracle_against_torch_fp32():
    """box_utils.decode + the scale multiply in torch fp32 (the reference's arithmetic) within the bar; past expf's
    overflow the fp32 sequence gives inf / NaN where the reference does."""
    rng = np.random.default_rng(1)
    h, w = 130, 97
    pri = post64.priors(h, w)
    loc = (rng.standard_normal((pri.shape[0], 4)) * 4).astype(np.float32)
    lt, pt = torch.from_numpy(loc), torch.from_numpy(pri)
    boxes = torch.cat((pt[:, :2] + lt[:, :2] * 0.1 * pt[:, 2:], pt[:, 2:] * torch.exp(lt[:, 2:] * 0.2)), 1)
    boxes[:, :2] -= boxes[:, 2:] / 2
    boxes[:, 2:] += boxes[:, :2]
    boxes = (boxes * torch.tensor([w, h, w, h], dtype=torch.float32)).numpy()
    want, s = post64.decode(loc, pri, w, h, 1.0)
    assert ratio(boxes, want, s).max() <= T['decode']
    big = loc[:4].copy()
    big[:, 2] = [440.0, 445.0, 1e4, np.inf]                        # 0.2 * l past ln(FLT_MAX) = 88.72
    f = post64.decode_f32(big, pri[:4], w, h, 1.0)
    assert np.isneginf(f[:, 0]).all() and np.isposinf(f[0, 2])      # exp(88) is finite, the box overflows at * w
    assert np.isnan(f[1:, 2]).all()                                # exp overflows: x2 = inf + -inf


def _py_cpu_nms(dets, thresh):
    """FaceBoxes/utils/nms/py_cpu_nms.py:10-38 as written there."""
    x1, y1, x2, y2, scores = dets[:, 0], dets[:, 1], dets[:, 2], dets[:, 3], dets[:, 4]
    areas = (x2 - x1 + 1) * (y2 - y1 + 1)
    order = scores.argsort()[::-1]
    keep = []
    with np.errstate(all='ignore'):
        while order.size > 0:
            i = order[0]
            keep.append(int(i))
            xx1, yy1 = np.maximum(x1[i], x1[order[1:]]), np.maximum(y1[i], y1[order[1:]])
            xx2, yy2 = np.minimum(x2[i], x2[order[1:]]), np.minimum(y2[i], y2[order[1:]])
            w, h = np.maximum(0.0, xx2 - xx1 + 1), np.maximum(0.0, yy2 - yy1 + 1)
            inter = w * h
            ovr = inter / (areas[i] + areas[order[1:]] - inter)
            order = order[np.where(ovr <= thresh)[0] + 1]
    return keep


def test_nms_on_nonfinite_boxes_equals_numpy():
    """The kernels' bit-matrix algorithm (render_emul.cpp, compiled from render_math.h) and the C port equal numpy's
    py_cpu_nms on boxes with NaN / inf coordinates: a NaN overlap fails `ovr <= thresh`, so py_cpu_nms drops the box."""
    out = os.path.join(tempfile.mkdtemp(prefix='post_emul_'), 'librender_emul.so')
    subprocess.run(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', out, os.path.join(HERE, 'host_emul', 'render_emul.cpp')],
                   check=True, capture_output=True)
    emul = C.CDLL(out)
    emul.emul_nms.restype = C.c_int
    ex = np.array([[0, 0, 10, 10, 0.9], [-np.inf, 0, np.nan, 10, 0.8], [1, 1, 11, 11, 0.7], [50, 50, 60, 60, 0.6]], np.float32)
    cases = [ex] + [post64.nms_cases(n, s) for s, n in enumerate((7, 64, 65, 200, 700))]
    for d in cases:
        order = d[:, 4].argsort()[::-1]
        ds = np.ascontiguousarray(d[order])
        keep = np.zeros(len(d), np.int32)
        for thr in (0.3, 0.5):
            want = _py_cpu_nms(d, np.float32(thr))
            assert render_port.py_cpu_nms(d, np.float32(thr)) == want
            assert render_port.cpu_nms(d, thr, ge=False) == want
            k = emul.emul_nms(ds.ctypes.data_as(C.c_void_p), len(d), C.c_double(thr), 0, keep.ctypes.data_as(C.c_void_p))
            assert order[keep[:k]].tolist() == want
            k = emul.emul_nms(ds.ctypes.data_as(C.c_void_p), len(d), C.c_double(thr), 1, keep.ctypes.data_as(C.c_void_p))
            assert order[keep[:k]].tolist() == render_port.cpu_nms(d, thr, ge=True)
    assert _py_cpu_nms(ex, 0.3) == [0, 3] and render_port.cpu_nms(ex, 0.3, ge=True) == [0, 1, 3]


def test_loss_oracles_against_reference():
    rng = np.random.default_rng(2)
    pred = torch.from_numpy(rng.standard_normal((6, 3, 68)).astype(np.float32) * 12)
    tg = torch.from_numpy(rng.standard_normal((6, 3, 68)).astype(np.float32) * 12)
    # the reference flattens (B,3,N) -> (B,3N) point-major; the mean does not depend on the order
    want, s = post64.wing_loss(pred.numpy(), tg.numpy())
    assert ratio(np.float64(rp.wing_loss(pred, tg)), want, s) <= T['wing']
    nan = tg.clone()
    nan[0, 0, :5] = float('nan')
    nan[1, 2, 3] = float('inf')
    want, s = post64.wing_loss(pred.numpy(), nan.numpy())
    got = float(rp.wing_loss(pred, nan))
    assert math.isinf(got) and math.isinf(want)                       # an inf delta is d >= omega
    nan[1, 2, 3] = 0.0
    want, s = post64.wing_loss(pred.numpy(), nan.numpy())
    assert np.isfinite(want) and ratio(np.float64(rp.wing_loss(pred, nan)), want, s) <= T['wing']
    all_nan = torch.full_like(tg, float('nan'))
    assert np.isnan(post64.wing_loss(pred.numpy(), all_nan.numpy())[0]) and math.isnan(float(rp.wing_loss(pred, all_nan)))
    p, q = (torch.from_numpy(rng.standard_normal((40, 62)).astype(np.float32) * 3) for _ in range(2))
    for mode, name in ((0, 'normal'), (1, 'only_3dmm')):
        want, s = post64.param_loss(p.numpy(), q.numpy(), mode)
        assert ratio(rp.param_loss(p, q, name).numpy(), want, s).max() <= T['param_loss']
