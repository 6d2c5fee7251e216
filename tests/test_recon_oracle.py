"""CPU checks of the float64 reconstruction oracle (oracle/recon64.py), its plan chooser, the wide and stress morphable
models used by tests/test_gpu_recon.py, and -- as a negative control -- a numpy emulation of the tensor-core kernels'
arithmetic, which must pass the bar and must fail it when any part of the scheme is left out."""
import numpy as np
import pytest

from oracle import recon64, synth_model
from oracle import reference_port as rp
from oracle.recon64 import magnitude_params, random_params, roi_rows
from oracle.stage_check import TAU, WIDE
from synergynet_b200 import synthetic

NOISE = 4e-6               # the fp32 reference (numpy sgemm, K = 50) against the float64 oracle, in units of S
F32, F16 = np.float32, np.float16


@pytest.fixture(scope='module')
def base3dmm():
    return synthetic.make_3dmm(0)


@pytest.fixture(scope='module')
def packs(base3dmm):
    return {'synthetic': synth_model.recon_pack(base3dmm),
            'wide': synth_model.recon_pack(synth_model.reparametrize_3dmm(base3dmm, **WIDE['recon64'])),
            'stress': synth_model.recon_pack(synth_model.stress_3dmm(base3dmm))}


def _inputs(pack):
    p_in, w_in = magnitude_params(pack, False)
    p_out, w_out = magnitude_params(pack, True)
    return [(random_params(16, 3), True), (p_in, w_in), (p_out, w_out)]


@pytest.mark.parametrize('model', ['synthetic', 'wide', 'stress'])
def test_oracle_agrees_with_fp32_reference(packs, model):
    pack = packs[model]
    for params, whitening in _inputs(pack):
        for dense in (False, True):
            for transform in (True, False):
                want, s = recon64.reconstruct(params[:6] if dense else params, pack, dense, whitening, transform)
                ref = rp.reconstruct_vertex_62(params[:6] if dense else params, pack, whitening, dense, transform)
                r, ix = recon64.worst(ref, want, s)
                assert r < NOISE, (model, dense, whitening, transform, r, ix)


def test_reparametrized_model_is_bit_identical(base3dmm):
    wide = synth_model.reparametrize_3dmm(base3dmm, **WIDE['recon64'])
    a, b = synth_model.recon_pack(base3dmm), synth_model.recon_pack(wide)
    assert not np.array_equal(recon64.ascale(a['param_mean'], a['param_std']),
                              recon64.ascale(b['param_mean'], b['param_std']))
    e = np.log2(recon64.ascale(b['param_mean'], b['param_std']) / recon64.ascale(a['param_mean'], a['param_std']))
    assert e.min() == WIDE['recon64']['lo'] and e.max() == WIDE['recon64']['hi']
    p = random_params(8, 4, 2.0)
    for dense in (False, True):
        assert np.array_equal(rp.reconstruct_vertex_62(p, a, True, dense), rp.reconstruct_vertex_62(p, b, True, dense))
        # raw coefficients of the reparametrized model are alpha_k / 2^e_k (exactly the de-whitened values)
        raw_a, raw_b = [(p * m['param_std'][:62] + m['param_mean'][:62]).astype(np.float32) for m in (a, b)]
        assert np.array_equal(rp.reconstruct_vertex_62(raw_a, a, False, dense),
                              rp.reconstruct_vertex_62(raw_b, b, False, dense))


def test_stress_model_has_the_special_rows(base3dmm):
    st = synth_model.recon_pack(synth_model.stress_3dmm(base3dmm))
    for dense in (False, True):
        u, w = recon64.basis_rows(st, dense)
        assert (u == 0).any() and (np.abs(w).max(1) == 0).any()
        m = np.abs(w).max(1)
        assert ((m > 2.0 ** 15) & (np.sort(np.abs(w), 1)[:, -2] < m * 2.0 ** -14)).any()
    k = synth_model.STRESS_ZERO_COEF
    assert recon64.ascale(st['param_mean'], st['param_std'])[k] == 2.0 ** 10


@pytest.mark.parametrize('sms', [114, 132])
def test_plan_chooser_covers_every_kind(sms):
    for kind, (batch, n_vert) in recon64.choose_dense_cases(sms).items():
        recon64.check_dense_case(kind, batch, n_vert, sms)
        assert batch * 3 * n_vert * 4 < 200e6 or n_vert == synthetic.NVER, kind
    for kind, (batch, n_pts) in recon64.choose_sparse_cases(sms).items():
        recon64.check_sparse_case(kind, batch, n_pts, sms)
        assert batch * 3 * n_pts * 4 < 200e6, kind
    assert recon64.dense_plan(64 * (sms // 2 + 1) - 5, sms, synthetic.NVER)['bands'] == 1
    # a one-item band and a short last band, computed by hand: 5 vertex tiles over 4 bands of 2 -> the last band has
    # one item and one band is idle
    assert recon64.dense_plan(10, 4, 5 * 128) == dict(ftiles=1, vtiles=5, bands=4, band_len=2, grid=4, idle=1,
                                                        last_band=1)


# ---- negative control: the kernels' arithmetic in numpy ----------------------------------------------------------------

def _split(x):
    hi = x.astype(F16)
    return hi, (x - hi.astype(F32)).astype(F16)


def _fma(a, b, c):
    return (a.astype(np.float64) * b + c).astype(F32)


def emulate_tc(params, pack, dense, whitening, transform=True, roi5=None, drop=None, clamp=False):
    """dense_alpha_kernel + the epilogue of dense_recon_{tc,fm}_kernel: fp16 hi / lo splits of the scaled coefficients
    and basis rows, the passes hi*hi, hi*lo, lo*hi (``drop`` one of them), the face scale (``clamp``: none, values
    clamped at 60000 as the split does), the fp32 epilogue."""
    mean, std = pack['param_mean'], pack['param_std']
    u, w = recon64.basis_rows(pack, dense)
    asc = recon64.ascale(mean, std).astype(F32)
    p32 = np.asarray(recon64.dewhiten(params, mean, std, whitening)[0], F32)
    a = p32[:, 12:62] * asc
    if clamp:
        fs = np.ones(len(a), F32)
        a = np.clip(a, -recon64.CLAMP, recon64.CLAMP).astype(F32)
    else:
        fs = recon64.face_scales(params, mean, std, whitening).astype(F32)
        a = a / fs[:, None]
    ah, al = _split(a)
    rs = recon64.row_scales(w, asc).astype(F32)
    wh, wl = _split((w / asc) * rs[:, None])
    terms = {'hh': (wh, ah), 'hl': (wh, al), 'lh': (wl, ah)}
    acc = sum(x.astype(np.float64) @ y.astype(np.float64).T for k, (x, y) in terms.items() if k != drop).astype(F32)
    b, n = len(params), len(u) // 3
    X = _fma(acc.T * fs[:, None], (1 / rs)[None, :].astype(F32), u[None, :]).reshape(b, n, 3)
    R = p32[:, :12].reshape(b, 3, 4)
    v = np.empty((b, 3, n), F32)
    for i in range(3):
        t = _fma(R[:, i, 2:3], X[:, :, 2], R[:, i, 3:4])
        t = _fma(R[:, i, 1:2], X[:, :, 1], t)
        v[:, i] = _fma(R[:, i, 0:1], X[:, :, 0], t)
    if transform or roi5 is not None:
        v[:, 1] = F32(121) - v[:, 1]
    if roi5 is not None:
        r = roi5.astype(F32)
        v[:, 0] = v[:, 0] * r[:, 0:1] + r[:, 1:2]
        v[:, 1] = v[:, 1] * r[:, 2:3] + r[:, 3:4]
        v[:, 2] = v[:, 2] * r[:, 4:5]
    return v


@pytest.mark.parametrize('model', ['synthetic', 'wide', 'stress'])
def test_emulated_kernel_passes_and_broken_ones_fail(packs, model):
    pack = packs[model]
    for params, whitening in _inputs(pack):
        for dense in (False, True):
            roi = roi_rows(len(params), 1) if whitening else None
            want = recon64.reconstruct(params, pack, dense, whitening, roi5=roi)
            r, ix = recon64.worst(emulate_tc(params, pack, dense, whitening, roi5=roi), *want)
            assert r < TAU['recon64']['tc'], (model, dense, r, ix)
            for drop in ('hh', 'hl', 'lh'):
                bad, _ = recon64.worst(emulate_tc(params, pack, dense, whitening, roi5=roi, drop=drop), *want)
                assert bad > 10 * TAU['recon64']['tc'], (model, dense, drop, bad)
            if np.any(recon64.face_scales(params, pack['param_mean'], pack['param_std'], whitening) > 1):
                bad, _ = recon64.worst(emulate_tc(params, pack, dense, whitening, roi5=roi, clamp=True), *want)
                assert bad > 10 * TAU['recon64']['tc'], (model, dense, 'clamp', bad)
