"""Every backbone stage of the three engines against the float64 oracle (oracle/block64.py), element by element.

Each stage is fed the GPU's own output of the previous stage, so errors do not accumulate and every element of every
stage is held to |got - want| <= TAU * S, S being the stage's first-order error scale.  The unfused engines are checked
conv by conv (52 convs), the fused engine block by block (17 blocks, conv index 3b - 1); then the pooled feature and
the 62 params.  The batches come from the device's SM count and cover every tile plan of the fused kernels
(oracle/tile_cover.py); the faces checked cover every tile kind of those plans.  H100 only.
"""
import pytest
import torch

from oracle import stage_check, synth_model, tile_cover
from oracle import reference_port as rp
from oracle.stage_check import (ENGINES, TOL, WIDE, make_model as _make_model, report as _report, seeded_crops,
                                stage_ratios, tau as _tau)
from synergynet_b200 import _lib, synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def sd_wide(sd):
    return synth_model.reparametrize_streams(sd, **WIDE['block64'])


@pytest.fixture(scope='module')
def model(synth_pack, sd):
    return _make_model(sd)


@pytest.fixture(scope='module')
def model_wide(synth_pack, sd_wide):
    return _make_model(sd_wide)


@pytest.fixture(scope='module')
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _engine(model, kind):
    model.set_engine(kind)
    return model._engine(torch.device('cuda', 0))


def _batch(sms, kind):
    batch = tile_cover.choose_batches(sms)[kind]
    tile_cover.check_plan(kind, batch, sms)
    return seeded_crops(batch, 900 + batch), tile_cover.faces_to_check(batch, sms, seed=batch)


@pytest.mark.parametrize('plan', ['mixed_pairs', 'odd_pairs', 'ragged_quads'])
@pytest.mark.parametrize('engine', list(ENGINES))
def test_every_stage_matches_float64_oracle(model, sd, sms, engine, plan):
    x, faces = _batch(sms, plan)
    eng = _engine(model, ENGINES[engine])
    try:
        ratios = stage_ratios(eng, engine == 'tc_fused', sd, x, faces)
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)
    _report(f'{engine} B={x.shape[0]} {plan} faces={len(faces)}', ratios)
    bad = stage_check.over(engine, ratios)
    assert not bad, bad


def test_single_pass_engine_fails_the_bar(model, sd, sms):
    """The one-pass fp16 engine drops the lo products and is otherwise identical: the per-element bar must see it at
    every fused block and at the tail, by a wide margin."""
    x, faces = _batch(sms, 'mixed_pairs')
    eng = _engine(model, _lib.ENGINE_TC_FUSED_1PASS)
    try:
        ratios = stage_ratios(eng, True, sd, x, faces)
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)
    _report(f'tc_fused_1pass B={x.shape[0]}', ratios)
    weak = {k: v for k, v in ratios.items() if k != 'params' and v[0] < 10 * _tau('tc_fused', k)}
    assert not weak, weak


@pytest.mark.parametrize('engine', list(ENGINES))
def test_rescaled_checkpoint_matches_golden(model_wide, engine):
    """The rescaled checkpoint computes the same function: its params and landmarks match the reference's vectors of
    the original checkpoint, and no block input leaves the range of the split-fp16 engines."""
    from golden.vectors import load_ref_vectors
    gold = load_ref_vectors()
    x = synthetic.normalize_crops(torch.from_numpy(gold['x_u8'])).cuda()
    eng = _engine(model_wide, ENGINES[engine])
    try:
        params = model_wide.forward_test(x)
        lmk = model_wide.reconstruct_vertex_62(params)
        assert eng.poll_saturation(warn=False) == 0
    finally:
        model_wide.set_engine(_lib.ENGINE_TC_FUSED)
    e_p = rp.max_rel_err(params.cpu().numpy(), gold['params'])
    e_l = rp.max_rel_err(lmk.cpu().numpy(), gold['lmk'])
    print(f'\n[{engine} rescaled] params err {e_p:.3e}  lmk err {e_l:.3e}')
    assert e_p < TOL and e_l < TOL


@pytest.mark.parametrize('engine', list(ENGINES))
def test_rescaled_checkpoint_every_stage(model_wide, sd_wide, sms, engine):
    x, faces = _batch(sms, 'odd_pairs')
    eng = _engine(model_wide, ENGINES[engine])
    try:
        ratios = stage_ratios(eng, engine == 'tc_fused', sd_wide, x, faces)
    finally:
        model_wide.set_engine(_lib.ENGINE_TC_FUSED)
    _report(f'{engine} rescaled B={x.shape[0]} faces={len(faces)}', ratios)
    bad = stage_check.over(engine, ratios)
    assert not bad, bad
