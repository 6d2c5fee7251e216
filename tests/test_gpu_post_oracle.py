"""The kernels at the two ends of the path against oracle/post64.py, every element of every call held to TAU * S:
pose_decode_kernel (uniform SO(3) rotations with anisotropic and sheared rows, yaw sweeps through the gimbal lock, zero /
overflowing / underflowing rows; B = 1, 127, 128, 129, 4283 with and without a crop box), faceboxes_rank_decode_kernel
(loc past expf's overflow, top_k truncation, one image and a stack of frames), nms_mask_kernel / nms_scan_kernel
(both modes, NaN / inf boxes, through syn_nms and syn_nms_batch) and the two loss kernels (deltas at omega and one ulp
either side, NaN / inf deltas, 4096 faces x 204, ParamLoss over several CTAs).  Prints the worst ratio of each kind."""
import numpy as np
import pytest
import torch

from oracle import post64, render_port, stage_check, synth_model
from oracle.check64 import ratio
from oracle.stage_check import TAU
from synergynet_b200 import _lib, detect, inference

pytestmark = pytest.mark.gpu
T = TAU['post64']
WORST = {}


def _note(kind, r):
    r = float(np.max(r)) if np.size(r) else 0.0
    WORST[kind] = max(WORST.get(kind, 0.0), r)
    assert r <= T[kind], (kind, r, T[kind])


def teardown_module(_):
    print('\n[post64] ' + '  '.join(f'{k}: {v:.3e} (tau {T[k]:.1e})' for k, v in sorted(WORST.items())))


@pytest.fixture(scope='module')
def model(synth_pack):
    return stage_check.make_model(synth_model.build_state_dict(0))


@pytest.fixture(scope='module')
def eng(model):
    return model._engine(torch.device('cuda', 0))


@pytest.fixture(scope='module')
def whitening(model):
    return (model.param_mean.detach().cpu().numpy().astype(np.float32)[:62],
            model.param_std.detach().cpu().numpy().astype(np.float32)[:62])


def _same_class(got, want):
    """NaN where want is NaN, the same infinity where want is infinite, 0 where want is 0."""
    assert np.array_equal(np.isnan(got), np.isnan(want))
    inf = np.isinf(want)
    assert np.array_equal(got[inf], want[inf]) and np.array_equal(np.isinf(got), inf)


def _check_pose(eng, prm, roi, mean, std, acc=True):
    ang, t3d = eng.pose_decode(torch.from_numpy(prm).cuda(), None if roi is None else torch.from_numpy(roi).cuda())
    a, t = ang.cpu().numpy(), t3d.cpu().numpy()
    P = post64.pose_p(prm, mean, std)
    ws, ss = post64.pose_angles_seq(post64.pose_rotation_f32(P))
    _same_class(a, ws)
    assert (a[ws == 0] == 0).all()
    fin = np.isfinite(ws)
    _note('pose_seq', ratio(a[fin], ws[fin], ss[fin]))
    if acc:
        wa, sa = post64.pose_angles_acc(P)
        _note('pose', ratio(a, wa, sa))
    wt, st = post64.pose_t3d(P, roi)
    if roi is None:
        assert np.array_equal(t.view(np.int32), P[:, [3, 7, 11]].view(np.int32))
    else:
        _same_class(t, wt)
        fin = np.isfinite(wt)
        _note('t3d', ratio(t[fin], wt[fin], st[fin]))
    return a


def _rois(n, seed):
    rng = np.random.default_rng(seed)
    x0, y0 = rng.uniform(-50, 900, n), rng.uniform(-50, 600, n)
    sz = rng.uniform(20, 400, (n, 2))
    return inference.roi_affine([[x0[i], y0[i], x0[i] + sz[i, 0], y0[i] + sz[i, 1], 1.0] for i in range(n)])


def test_pose_so3_every_batch_shape(eng, whitening):
    mean, std = whitening
    prm = post64.pose_cases_so3(mean, std, 4283, seed=0)
    roi = _rois(4283, 1)
    for b in (1, 127, 128, 129, 4283):
        _check_pose(eng, prm[:b], None, mean, std)
        _check_pose(eng, prm[:b], roi[:b], mean, std)


def test_pose_yaw_sweep_through_the_lock(eng, whitening):
    """R20 on every fp32 value within 64 ulps of +-1, exactly +-1 and above 1: finite angles, the lock branch of R20's
    sign at |R20| >= 1."""
    mean, std = whitening
    prm, r20 = post64.pose_cases_lock(mean, std)
    a = _check_pose(eng, prm, _rois(len(prm), 2), mean, std)
    assert np.isfinite(a).all()
    lock = np.abs(r20) >= 1
    assert (np.abs(r20) > 1).any() and np.array_equal(a[lock, 0], np.where(r20[lock] > 0, -90.0, 90.0))


def test_pose_zero_overflow_underflow_rows(eng, model, whitening):
    """Camera rows set directly (identity whitening): NaN, inf and 0 exactly where numpy's fp32 sequence gives them."""
    mean, std = whitening
    P = post64.pose_cases_special()
    prm = np.zeros((P.shape[0], 62), np.float32)
    prm[:, :12] = P
    zero, one = np.zeros(62, np.float32), np.ones(62, np.float32)
    lib = eng._lib
    try:
        _lib.check(lib.syn_set_whitening(eng._h, zero.ctypes.data, one.ctypes.data))
        eng.commit()
        _check_pose(eng, prm, None, zero, one, acc=False)
        _check_pose(eng, prm, _rois(len(prm), 3), zero, one, acc=False)
    finally:
        _lib.check(lib.syn_set_whitening(eng._h, mean.ctypes.data, std.ctypes.data))
        eng.commit()


def _decode_cases(h, w, frames, seed):
    rng = np.random.default_rng(seed)
    npri = detect.num_priors(h, w)
    loc = (rng.standard_normal((frames, npri, 4)) * 3).astype(np.float32)
    big = rng.random((frames, npri)) < 0.05
    loc[..., 2][big] = rng.choice([300.0, 430.0, 440.0, 445.0, 1e4, np.inf], big.sum())   # 0.2 l past 88.72 from 445
    loc[..., 3][big] = rng.choice([-1e4, 100.0, 445.0, np.inf], big.sum())
    s = np.round(rng.uniform(0, 1, (frames, npri)) * 64) / 64                             # ties in the score order
    conf = np.stack([1 - s, s], -1).astype(np.float32)
    return loc, conf


def _check_decode(dets, n, loc, conf, h, w, k, thresh=0.05):
    order = post64.decode_order(conf, thresh, k)
    assert n == len(order)
    got = dets[:n]
    assert np.array_equal(got[:, 4], conf[order, 1])
    pri = post64.priors(h, w)[order]
    f32 = post64.decode_f32(loc[order], pri, w, h, 1.0)
    want, s = post64.decode(loc[order], pri, w, h, 1.0)
    _same_class(got[:, :4], f32)
    fin = np.isfinite(f32)
    _note('decode', ratio(got[:, :4][fin], want[fin], s[fin]))


def test_box_decode_overflow_and_top_k(eng):
    for (h, w), k in (((130, 97), 5000), ((130, 97), 40), ((300, 420), 700)):
        loc, conf = _decode_cases(h, w, 3, seed=h + k)
        for f in range(3):
            dets, n = detect.decode_device(torch.from_numpy(loc[f]).cuda(), torch.from_numpy(conf[f]).cuda(), h, w, k=k)
            _check_decode(dets.cpu().numpy(), int(n.item()), loc[f], conf[f], h, w, k)
        db, nb = detect.decode_batch_device(torch.from_numpy(loc).cuda(), torch.from_numpy(conf).cuda(), h, w, k=k)
        for f in range(3):
            _check_decode(db[f].cpu().numpy(), int(nb[f].item()), loc[f], conf[f], h, w, k)


def test_nms_nonfinite_boxes_both_modes(eng):
    """syn_nms and syn_nms_batch on boxes with NaN / inf coordinates and zero-overlap pairs: py_cpu_nms drops a NaN
    overlap (`ovr <= thresh` fails), cpu_nms keeps it (`ovr >= thresh` fails)."""
    dev = torch.device('cuda', 0)
    sizes = (4, 7, 64, 65, 200, 700)
    cases = [np.array([[0, 0, 10, 10, 0.9], [-np.inf, 0, np.nan, 10, 0.8], [1, 1, 11, 11, 0.7], [50, 50, 60, 60, 0.6]],
                      np.float32)] + [post64.nms_cases(n, 10 + n) for n in sizes[1:]]
    rows = max(sizes)
    for thr in (0.3, 0.5):
        for mode, want_fn in ((_lib.NMS_PY_CPU_NMS, lambda d: render_port.py_cpu_nms(d, np.float32(thr))),
                              (_lib.NMS_CPU_NMS, lambda d: render_port.cpu_nms(d, thr, ge=True))):
            stack = np.zeros((len(cases), rows, 5), np.float32)
            counts = []
            for f, d in enumerate(cases):
                order = d[:, 4].argsort()[::-1]
                keep, nk = detect.nms_device(torch.from_numpy(np.ascontiguousarray(d[order])).to(dev), thr, mode)
                assert order[keep[:int(nk.item())].cpu().numpy()].tolist() == want_fn(d), (mode, thr, len(d))
                stack[f, :len(d)] = d[order]
                counts.append(len(d))
            kb, nkb = detect.nms_batch_device(torch.from_numpy(stack).to(dev), torch.tensor(counts, dtype=torch.int32, device=dev),
                                              thr, mode)
            for f, d in enumerate(cases):
                order = d[:, 4].argsort()[::-1]
                assert order[kb[f, :int(nkb[f].item())].cpu().numpy()].tolist() == want_fn(d), (mode, thr, f)
    assert detect.py_cpu_nms(cases[0], 0.3) == [0, 3] and detect.cpu_nms(cases[0], 0.3) == [0, 1, 3]


def test_wing_loss_edges_and_size(eng):
    rng = np.random.default_rng(5)
    om = np.float32(10)
    for faces in (1, 37, 4096):
        pred = (rng.standard_normal((faces, 3, 68)) * 12).astype(np.float32)
        tg = (rng.standard_normal((faces, 3, 68)) * 12).astype(np.float32)
        flat_p, flat_t = pred.reshape(-1), tg.reshape(-1)
        flat_p[:6] = 0
        flat_t[:6] = [om, np.nextafter(om, np.float32(0)), np.nextafter(om, np.float32(20)), -om,
                      -np.nextafter(om, np.float32(0)), -np.nextafter(om, np.float32(20))]
        for variant in ('plain', 'nan', 'inf', 'all_nan'):
            p, t = pred.copy(), tg.copy()
            if variant == 'nan':
                t.reshape(-1)[rng.choice(t.size, max(1, t.size // 50), replace=False)] = np.nan
                p.reshape(-1)[7] = t.reshape(-1)[7] = np.inf               # inf - inf: a NaN delta
            elif variant == 'inf':
                t.reshape(-1)[9] = -np.inf
            elif variant == 'all_nan':
                t[:] = np.nan
            got = np.asarray(float(eng.wing_loss(torch.from_numpy(p).cuda(), torch.from_numpy(t).cuda()).cpu()))
            want, s = post64.wing_loss(p, t)
            _same_class(got, want)
            if np.isfinite(want):
                _note('wing', ratio(got, want, s))


def test_param_loss_several_ctas(eng):
    rng = np.random.default_rng(6)
    for b in (1, 300):
        p = (rng.standard_normal((b, 62)) * 10.0 ** rng.uniform(-3, 2, (b, 1))).astype(np.float32)
        q = (p + rng.standard_normal((b, 62)) * 10.0 ** rng.uniform(-4, 1, (b, 1))).astype(np.float32)
        q[0, :12] = p[0, :12]                                             # one sample with an exact first mean
        for mode, name in ((0, 'normal'), (1, 'only_3dmm')):
            got = eng.param_loss(torch.from_numpy(p).cuda(), torch.from_numpy(q).cuda(), mode=name).cpu().numpy()
            want, s = post64.param_loss(p, q, mode)
            _note('param_loss', ratio(got, want, s))
