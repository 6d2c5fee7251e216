"""The 3DMM reconstruction (landmarks, dense mesh, image-space mesh) against the float64 oracle (oracle/recon64.py),
element by element: every element of every call is held to |got - want| <= TAU * S.

The cases cover the work plans of both tensor-core kernels (oracle/recon64.py choose_*_cases, derived from the SM count),
output rows on every 4-byte phase, outputs at every float offset from an aligned buffer, batches far larger than the
oracle can check (by position invariance against an oracle-checked pool of faces), coefficients from the mean to far
beyond the fp16 range of the split, and the state changes that re-pack the basis.  H100 only.
"""
import numpy as np
import pytest
import torch

from oracle import recon64, synth_model
from oracle.recon64 import magnitude_params, random_params, roi_rows
from oracle.stage_check import TAU, WIDE, Ratios, report as print_report
from synergynet_b200 import _lib, synthetic

pytestmark = pytest.mark.gpu

PATH = {_lib.ENGINE_SIMT_FP32: 'fp32', _lib.ENGINE_TC_FUSED: 'tc'}
RATIOS = Ratios()


def check(tag, path, got, want_s):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    r, ix = RATIOS.add(path, f'{path} {tag}', got, want_s)
    assert r <= TAU['recon64'][path], f'{tag} ({path}): |got - want| / S = {r:.3e} at {ix}'


@pytest.fixture(scope='module', autouse=True)
def report():
    yield
    print_report('reconstruction', RATIOS)


# ---- inputs ---------------------------------------------------------------------------------------------------------

def raw(params, pack):
    """The de-whitened fp32 parameters (to call with whitening off)."""
    return (params * pack['param_std'][:62] + pack['param_mean'][:62]).astype(np.float32)


# ---- fixtures -------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def base3dmm():
    return synthetic.make_3dmm(0)


@pytest.fixture(scope='module')
def prod(base3dmm):
    return synth_model.recon_pack(base3dmm)


@pytest.fixture(scope='module')
def eng(synth_pack):
    from synergynet_b200.engine import Engine
    e = Engine(0)
    e.load_backbone(synth_model.build_state_dict(0))
    e.set_engine(_lib.ENGINE_TC_FUSED)
    e.loaded = None
    yield e
    e.close()


def use(eng, pack, engine=_lib.ENGINE_TC_FUSED):
    """Load ``pack`` into the engine (once) and select the engine kind."""
    if eng.loaded is not pack:
        eng.load_3dmm(pack['param_mean'], pack['param_std'], pack['u_base'], pack['w_shp_base'], pack['w_exp_base'],
                      pack['u'], pack['w_shp'], pack['w_exp'])
        eng.commit()
        eng.loaded = pack
    eng.set_engine(engine)
    return eng


def recon(eng, params, dense, whitening=True, transform=True):
    return eng.reconstruct(torch.from_numpy(params).cuda(), dense=dense, whitening=whitening, transform=transform)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


_oracle_cache = {}


def oracle(pack, params, dense, whitening=True, transform=True, roi5=None, key=None):
    k = None if key is None else (key, dense, whitening, transform, roi5 is not None)
    if k is not None and k in _oracle_cache:
        return _oracle_cache[k]
    out = recon64.reconstruct_chunked(params, pack, dense=dense, whitening=whitening, transform=transform, roi5=roi5)
    if k is not None:
        _oracle_cache[k] = out
    return out


# ---- flags, entry points and engines --------------------------------------------------------------------------------

@pytest.mark.parametrize('engine', [_lib.ENGINE_SIMT_FP32, _lib.ENGINE_TC_FUSED], ids=['engine0', 'engine2'])
def test_flags_and_entry_points(eng, prod, engine):
    use(eng, prod, engine)
    wp = random_params(70, 1)
    rp_ = raw(wp, prod)
    for dense in (False, True):
        for whitening in (True, False):
            for transform in (True, False):
                p = wp if whitening else rp_
                got = recon(eng, p, dense, whitening, transform)
                want = oracle(prod, p, dense, whitening, transform, key=('flags', whitening))
                check(f'{"dense" if dense else "sparse"} w{int(whitening)} t{int(transform)}', PATH[engine], got, want)
        roi = roi_rows(70, 2)
        got = eng.reconstruct_image(torch.from_numpy(wp).cuda(), torch.from_numpy(roi).cuda(), dense=dense)
        check(f'{"dense" if dense else "sparse"} image', 'tc', got, oracle(prod, wp, dense, roi5=roi))
    assert eng.poll_error() == 0


def test_engines_1_and_3_reconstruct_like_engine_2(eng, prod):
    wp = random_params(70, 3)
    want = {}
    for kind in (_lib.ENGINE_TC_FUSED, _lib.ENGINE_TC_BF16X3, _lib.ENGINE_TC_FUSED_1PASS):
        use(eng, prod, kind)
        got = [recon(eng, wp, d) for d in (False, True)]
        if not want:
            want = got
        assert all(torch.equal(a, b) for a, b in zip(got, want)), kind
    use(eng, prod)


# ---- dense work plans and row phases --------------------------------------------------------------------------------

def narrow_pack(base3dmm, n_vert, seed):
    return synth_model.recon_pack(base3dmm, dense=synth_model.basis_arrays(n_vert, seed))


@pytest.mark.parametrize('kind', ['small_idle', 'ragged_multi', 'short_last', 'one_item', 'one_band', 'grid_gt_sms'])
def test_dense_plan_kinds(eng, base3dmm, prod, kind):
    batch, n_vert = recon64.choose_dense_cases(sms())[kind]
    recon64.check_dense_case(kind, batch, n_vert, sms())
    pack = prod if n_vert == synthetic.NVER else narrow_pack(base3dmm, n_vert, 20 + n_vert)
    use(eng, pack)
    p = random_params(batch, 30 + batch)
    got = recon(eng, p, True).cpu().numpy()
    check(f'dense plan {kind}', 'tc', got, oracle(pack, p, True))
    assert eng.poll_error() == 0


@pytest.mark.parametrize('n_vert', [1, 5, 8 * 37, 127, 128, 129])
def test_dense_rows_on_every_phase(eng, base3dmm, n_vert):
    """Rows of n_vert floats start on every 4-byte phase of a sector (on phase 0 only when 8 divides n_vert); with
    B = 200 the last face tile is ragged."""
    pack = narrow_pack(base3dmm, n_vert, 40 + n_vert)
    use(eng, pack)
    p = random_params(200, 50 + n_vert)
    check(f'dense n_vert {n_vert}', 'tc', recon(eng, p, True), oracle(pack, p, True))
    roi = roi_rows(200, 3)
    got = eng.reconstruct_image(torch.from_numpy(p).cuda(), torch.from_numpy(roi).cuda(), dense=True)
    check(f'dense image n_vert {n_vert}', 'tc', got, oracle(pack, p, True, roi5=roi))


# ---- output alignment ------------------------------------------------------------------------------------------------

GUARD = 256
SENTINEL = 0x7FBADBAD                      # a NaN no kernel writes


@pytest.mark.parametrize('case', ['prod128', 'narrow129', 'image'])
def test_output_at_every_float_offset(eng, base3dmm, prod, case):
    """``out = buf + off`` for off = 0..7 floats: the guard bands on both sides stay untouched and every offset gives
    the same bits as off = 0."""
    pack = narrow_pack(base3dmm, 129, 7) if case == 'narrow129' else prod
    use(eng, pack)
    batch = 128 if case == 'prod128' else 70
    n = pack['u'].size // 3
    p = torch.from_numpy(random_params(batch, 60)).cuda()
    roi = torch.from_numpy(roi_rows(batch, 61)).cuda()
    size = batch * 3 * n
    lib, st = eng._lib, torch.cuda.current_stream().cuda_stream
    ref = None
    for off in range(8):
        buf = torch.full((GUARD + off + size + GUARD,), SENTINEL, dtype=torch.int32, device='cuda')
        ptr = buf.data_ptr() + 4 * (GUARD + off)
        if case == 'image':
            _lib.check(lib.syn_reconstruct_image(eng._h, p.data_ptr(), batch, 1, roi.data_ptr(), ptr, st))
        else:
            _lib.check(lib.syn_reconstruct(eng._h, p.data_ptr(), batch, 1, 1, 1, ptr, st))
        torch.cuda.synchronize()
        assert bool((buf[:GUARD + off] == SENTINEL).all()) and bool((buf[GUARD + off + size:] == SENTINEL).all()), off
        out = buf[GUARD + off:GUARD + off + size].clone()
        if ref is None:
            ref = out
            want = oracle(pack, p.cpu().numpy(), True, roi5=roi.cpu().numpy() if case == 'image' else None)
            check(f'dense offsets {case}', 'tc', out.view(torch.float32).view(batch, 3, n), want)
        assert torch.equal(out, ref), off


# ---- large batches: position invariance -----------------------------------------------------------------------------

def test_large_dense_batch_position_invariance(eng, prod):
    """A pool of 64 distinct faces is checked against the oracle; then a batch with one vertex band per face tile
    (B ~ 64 (SMs / 2 + 1), 2.7 GB of output) places pool face (slot + tile) % 64 at every face-in-tile slot -- so
    every pool face takes every slot, team, sub-round and row phase -- and each face must equal its pool result bit for
    bit."""
    use(eng, prod)
    pool = random_params(64, 70)
    ref = recon(eng, pool, True)
    check('dense pool', 'tc', ref, oracle(prod, pool, True))
    batch = 64 * (sms() // 2 + 1) - 5
    plan = recon64.dense_plan(batch, sms(), synthetic.NVER)
    assert plan['bands'] == 1 and plan['ftiles'] * 64 > batch, plan
    b = torch.arange(batch, device='cuda')
    perm = (b + b // 64) % 64
    out = eng.reconstruct(torch.from_numpy(pool).cuda()[perm], dense=True)
    for c in range(0, batch, 512):
        assert torch.equal(out[c:c + 512], ref[perm[c:c + 512]]), c
    del out
    assert eng.poll_error() == 0


# ---- sparse work plans ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind', ['ring_wrap', 'tile_cross', 'meta_cycle'])
def test_sparse_plan_kinds(eng, base3dmm, prod, kind):
    batch, n_pts = recon64.choose_sparse_cases(sms())[kind]
    recon64.check_sparse_case(kind, batch, n_pts, sms())
    pack = prod if n_pts == 68 else synth_model.recon_pack(base3dmm, sparse=synth_model.basis_arrays(n_pts, 80))
    use(eng, pack)
    p = random_params(batch, 90)
    want = oracle(pack, p, False) if batch <= 4096 else recon64.reconstruct(p, pack, dense=False)
    check(f'sparse plan {kind}', 'tc', recon(eng, p, False), want)
    assert eng.poll_error() == 0


# ---- coefficient magnitudes -------------------------------------------------------------------------------------------

def _magnitude_case(eng, pack, beyond, engine, tag):
    use(eng, pack, engine)
    p, whitening = magnitude_params(pack, beyond)
    for dense in (False, True):
        got = recon(eng, p, dense, whitening)
        assert bool(torch.isfinite(got).all())
        check(f'{tag} {"dense" if dense else "sparse"}', PATH[engine], got, oracle(pack, p, dense, whitening))
    if whitening:
        roi = roi_rows(len(p), 9)
        got = eng.reconstruct_image(torch.from_numpy(p).cuda(), torch.from_numpy(roi).cuda(), dense=True)
        check(f'{tag} image', 'tc', got, oracle(pack, p, True, roi5=roi))
    use(eng, pack)


@pytest.fixture(scope='module')
def packs(base3dmm, prod):
    return {'synthetic': prod,
            'wide': synth_model.recon_pack(synth_model.reparametrize_3dmm(base3dmm, **WIDE['recon64'])),
            'stress': synth_model.recon_pack(synth_model.stress_3dmm(base3dmm))}


@pytest.mark.parametrize('engine', [_lib.ENGINE_SIMT_FP32, _lib.ENGINE_TC_FUSED], ids=['engine0', 'engine2'])
@pytest.mark.parametrize('model', ['synthetic', 'wide', 'stress'])
def test_coefficients_within_fp16_range(eng, packs, model, engine):
    _magnitude_case(eng, packs[model], False, engine, f'in range {model}')


@pytest.mark.parametrize('engine', [_lib.ENGINE_SIMT_FP32, _lib.ENGINE_TC_FUSED], ids=['engine0', 'engine2'])
@pytest.mark.parametrize('model', ['synthetic', 'wide', 'stress'])
def test_coefficients_beyond_fp16_range(eng, packs, model, engine):
    _magnitude_case(eng, packs[model], True, engine, f'beyond {model}')


@pytest.mark.parametrize('bad', [float('nan'), float('inf'), -float('inf')], ids=['nan', 'inf', '-inf'])
def test_nonfinite_coefficient_raises_the_flag(eng, prod, bad):
    """A NaN or +-Inf shape coefficient of one face reaches the fp16 split of dense_alpha_kernel: the call raises the
    saturation flag, and every other face of the batch (two face tiles) keeps the clean call's bits."""
    use(eng, prod)
    p = random_params(70, 91)
    clean = recon(eng, p, True).cpu()
    assert eng.poll_saturation(warn=False) == 0
    q = p.copy()
    q[65, 12 + 7] = bad
    got = recon(eng, q, True).cpu()
    assert eng.poll_saturation(warn=False) == 1
    assert eng.poll_saturation(warn=False) == 0
    keep = torch.arange(70) != 65
    assert torch.equal(got[keep].view(torch.int32), clean[keep].view(torch.int32))


# ---- state changes ----------------------------------------------------------------------------------------------------

def test_state_changes_are_picked_up(eng, base3dmm, prod):
    use(eng, prod)
    small, big = random_params(10, 100), random_params(5000, 101)
    first = [recon(eng, small, d) for d in (False, True)]
    recon(eng, big, False)
    recon(eng, big[:1100], True)                                  # the workspace grows
    again = [recon(eng, small, d) for d in (False, True)]
    assert all(torch.equal(a, b) for a, b in zip(first, again))
    # new whitening statistics: new alpha scales, the basis images are re-packed on commit
    pack = dict(prod)
    pack['param_std'] = prod['param_std'] * np.float32(16.0)
    pack['param_mean'] = prod['param_mean'] * np.float32(0.5)
    mean, std = torch.from_numpy(pack['param_mean'][:62].copy()), torch.from_numpy(pack['param_std'][:62].copy())
    _lib.check(eng._lib.syn_set_whitening(eng._h, mean.data_ptr(), std.data_ptr()))
    eng.commit()
    eng.loaded = pack
    for d in (False, True):
        check('new whitening', 'tc', recon(eng, small, d), oracle(pack, small, d))
    # a new dense basis alone
    u, ws, we = synth_model.basis_arrays(300, 110)
    _lib.check(eng._lib.syn_set_basis_dense(eng._h, u.ctypes.data, ws.ctypes.data, we.ctypes.data, 300))
    eng.commit()
    eng.n_vert = 300
    pack = dict(pack, u=u, w_shp=ws, w_exp=we)
    eng.loaded = pack
    check('new dense basis', 'tc', recon(eng, small, True), oracle(pack, small, True))
    check('new dense basis sparse', 'tc', recon(eng, small, False), oracle(pack, small, False))
    eng.loaded = None
    assert eng.poll_error() == 0
