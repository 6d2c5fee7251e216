"""The weight side of the split-fp16 engines' fixed-scale packers, against the float64 oracle (oracle/block64.py).
H100 only.

Expand spread.  One hidden channel of every block, 1-17, dead with its folded expand weights 2^k times the others'
(``synth_model.scale_hidden_channel``): what BN folding makes of a channel with a near-zero running variance.  In the
blocks with several hidden chunks the channel lies past the first chunk.  Engines 0-2 keep every stage under its bar
for k up to 100; the fused expand scaled its whole layer with the largest channel's power of two before, and failed.

Output-channel binades.  One output channel of every non-residual project conv (blocks 1, 2, 4, 7, 11, 14, 17: a skip
would hide the channel in S) and of features.18 (the tail) with its folded weights moved into binade 2^e
(``synth_model.scale_output_channel``).  Down to 2^-108 engines 0-2 pass the bar; below it the packers' capped scale
costs bits, and every output stays finite, no flag is raised and each stage stays within 4x the emulation's figure for
the binade (``oracle/pack_emul.binade_ratio``).

Zero channel.  An all-zero output channel with a bias returns exactly that bias on every engine.
"""
import math

import pytest
import torch

from oracle import pack_emul, stage_check, synth_model, tile_cover
from oracle.stage_check import make_model, report, seeded_crops, stage_ratios, tau
from synergynet_b200 import _lib
from synergynet_b200.backbone import conv_plan

pytestmark = pytest.mark.gpu

SPREADS = (0, 8, 11, 12, 14, 16, 20, 24, 40, 100)
BINADES = (2, 0, -40, -80, -100, -108, -112, -116, -118, -120, -122, -126, -130, -140, -149)
PROJECTS = [s.index for s in conv_plan() if s.kind == 'project' and not s.residual] + [len(conv_plan()) - 1]
ZERO_BIAS = 0.3125
ALL = (_lib.ENGINE_SIMT_FP32, _lib.ENGINE_TC_BF16X3, _lib.ENGINE_TC_FUSED, _lib.ENGINE_TC_FUSED_1PASS)


def _hidden(block: int) -> int:
    """The hidden channel scaled in a block: 5/7 of the way through, past the first chunk of every multi-chunk config
    (the largest chunk has 64 channels, the smallest multi-chunk block 96)."""
    hid = [s.cout for s in conv_plan() if s.block == block and s.kind in ('stem', 'expand', 'dw')][-1]
    return hid * 5 // 7


@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def batch():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    b = tile_cover.choose_batches(sms)['odd_pairs']
    tile_cover.check_plan('odd_pairs', b, sms)
    return seeded_crops(b, 900 + b), tile_cover.faces_to_check(b, sms, seed=b)


def _engine(model, kind):
    model.set_engine(kind)
    return model._engine(torch.device('cuda', 0))


_MODELS = {}


def _model(key, build):
    """One model per checkpoint, kept for the engines of the same parameter (the last one only)."""
    if key not in _MODELS:
        _MODELS.clear()
        sd_k = build()
        _MODELS[key] = (sd_k, make_model(sd_k))
    return _MODELS[key]


def _spread_sd(sd, k):
    for b in range(1, 18):
        sd = synth_model.scale_hidden_channel(sd, b, _hidden(b), 2.0 ** k)
    return sd


@pytest.mark.parametrize('engine', list(stage_check.ENGINES))
@pytest.mark.parametrize('k', SPREADS)
def test_expand_spread(synth_pack, sd, batch, k, engine):
    sd_k, model = _model(('spread', k), lambda: _spread_sd(sd, k))
    x, faces = batch
    try:
        ratios = stage_ratios(_engine(model, stage_check.ENGINES[engine]), engine == 'tc_fused', sd_k, x, faces)
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)
    report(f'{engine} expand spread 2^{k}', ratios)
    bad = stage_check.over(engine, ratios)
    assert not bad, bad


def _binade_sd(sd, e):
    for idx in PROJECTS:
        ch = conv_plan()[idx].cout * 3 // 5
        m = synth_model.channel_max(sd, idx, ch)
        sd = synth_model.scale_output_channel(sd, idx, ch, 2.0 ** (e - math.floor(math.log2(m))))
        assert 2.0 ** e <= synth_model.channel_max(sd, idx, ch) < 2.0 ** (e + 1), (idx, e)
    return sd


@pytest.fixture(scope='module')
def figures():
    """The emulation's worst ratio per binade below 2^-108."""
    return {e: pack_emul.binade_ratio(e) for e in BINADES if e <= pack_emul.CAP_FLOOR}


@pytest.mark.parametrize('engine', list(stage_check.ENGINES))
@pytest.mark.parametrize('e', BINADES)
def test_output_channel_binades(synth_pack, sd, batch, figures, e, engine):
    sd_e, model = _model(('binade', e), lambda: _binade_sd(sd, e))
    x, faces = batch
    eng = _engine(model, stage_check.ENGINES[engine])
    try:
        params, pool = eng.forward(x, want_pool=True)
        assert bool(torch.isfinite(params).all()) and bool(torch.isfinite(pool).all())
        ratios = stage_ratios(eng, engine == 'tc_fused', sd_e, x, faces)     # also: no error and no saturation flag
        if engine == 'tc_fused':
            for b in range(1, 18):
                assert bool(torch.isfinite(eng.debug_forward_until(x, 3 * b - 1)).all()), b
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)
    report(f'{engine} output channels at 2^{e}', ratios)
    assert all(math.isfinite(v[0]) for v in ratios.values()), ratios
    if e > pack_emul.CAP_FLOOR:
        bad = stage_check.over(engine, ratios)
    else:
        bad = {s: v for s, v in ratios.items() if v[0] > max(tau(engine, s), 4 * figures[e])}
    assert not bad, (e, figures.get(e), bad)


@pytest.mark.parametrize('kind', ALL)
def test_zero_channel_returns_its_bias(synth_pack, sd, batch, kind):
    """An all-zero output channel of every non-residual project conv and of the tail, with bias 0.3125: the block output
    (and, for the tail, the pooled feature after the ReLU6) holds exactly the bias at every pixel of every face."""
    def build():
        out = sd
        for idx in PROJECTS:
            out = synth_model.scale_output_channel(out, idx, conv_plan()[idx].cout // 3, 0.0, bias=ZERO_BIAS)
        return out
    _, model = _model('zero', build)
    x = batch[0]
    eng = _engine(model, kind)
    try:
        for idx in PROJECTS[:-1]:
            y = eng.debug_forward_until(x, idx)[..., conv_plan()[idx].cout // 3]
            assert torch.equal(y, torch.full_like(y, ZERO_BIAS)), (kind, idx)
        pool = eng.forward(x, want_pool=True)[1][:, conv_plan()[-1].cout // 3]
        assert torch.equal(pool, torch.full_like(pool, ZERO_BIAS)), kind
        assert eng.poll_error() == 0 and eng.poll_saturation(warn=False) == 0
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)
