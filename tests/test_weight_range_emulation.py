"""The fixed-scale weight packers of the split-fp16 engines (``oracle/pack_emul.py``, a numpy restatement) held to the
float64 oracle's S across channel spreads and weight binades, without a GPU.

The fused expand used to scale its whole layer by one power of two (``LAYER``): one hidden channel 2^k above the rest
pushes the others' weights down by 2^k in the fp16 split, and their lo halves into subnormals.  ``CHANNEL`` (the
packer's scheme now) scales each hidden channel on its own.  The per-channel packers cap the scale at 2^117, so a
channel whose max |w| is below 2^-108 packs under [256, 512) with fewer bits: finite, and what ``binade_ratio`` gives
per binade is the bound ``tests/test_gpu_weight_range.py`` holds the GPU to there.
"""
import numpy as np
import pytest

from oracle import pack_emul as pe
from oracle.stage_check import TAU

BAR = TAU['tc_bf16x3']['conv']                # the bar of one split-fp16 conv stage
SPREADS = (0, 8, 11, 12, 14, 16, 20, 24, 40, 100)
FIRST_FAIL = 16                               # where the layer-wide scale failed on the GPU too (block 3, 4.1e-7 of S)
BINADES = (2, 0, -40, -80, -100, -108, -112, -116, -118, -120, -122, -126, -130, -140, -149)
HOT = 7                                       # the hidden channel scaled by 2^k


def _expand_layer(k: int, seed: int = 0):
    """(block input (2048, 24), weights (24, 144) fp32, bias): Gaussian, hidden channel HOT 2^k above the rest."""
    rng = np.random.default_rng(seed)
    a = pe.f32(rng.standard_normal((2048, 24)))
    w = rng.standard_normal((24, 144)) / 24 ** 0.5
    w[:, HOT] *= 2.0 ** k
    return a, pe.f32(w), pe.f32(rng.standard_normal(144) * 0.1)


def _expand_worst(k: int, scheme: str) -> float:
    """The worst ratio over the hidden channels other than the scaled one."""
    a, w, b = _expand_layer(k)
    r = pe.ratios(pe.expand(a, w, b, scheme), a, w.astype(np.float64), b.astype(np.float64))
    return float(np.nan_to_num(np.delete(r, HOT, axis=1), nan=np.inf).max())


@pytest.mark.parametrize('k', SPREADS)
def test_expand_spread(k):
    """The layer-wide scale fails the bar from 2^16 on; the per-channel scale passes at every spread up to 2^100."""
    layer, channel = _expand_worst(k, pe.LAYER), _expand_worst(k, pe.CHANNEL)
    print(f'\n[spread 2^{k}] layer-wide {layer:.3e}  per channel {channel:.3e}')
    assert channel <= BAR, (k, channel)
    assert (layer > BAR) == (k >= FIRST_FAIL), (k, layer)


def test_schemes_agree_bit_for_bit_when_channel_maxima_share_a_binade():
    """Every channel maximum in the layer maximum's binade: both schemes pick the same scale and compute the same bits."""
    rng = np.random.default_rng(3)
    a = pe.f32(rng.standard_normal((512, 32)) * 4)
    w = rng.uniform(-1.0, 1.0, (32, 96))
    w[rng.integers(0, 32, 96), np.arange(96)] = rng.uniform(1.0, 2.0, 96) * np.where(rng.random(96) < 0.5, -1, 1)
    w = pe.f32(w * 2.0 ** -3)
    b = pe.f32(rng.standard_normal(96))
    assert (pe.scale_exp(np.abs(w).max(axis=0)) == pe.scale_exp(np.abs(w).max())).all()
    got = [pe.expand(a, w, b, s) for s in (pe.LAYER, pe.CHANNEL)]
    assert np.array_equal(got[0].view(np.int64), got[1].view(np.int64))


def test_per_channel_binade_sweep():
    """Down to 2^-108 the per-channel packers pass the bar; below it the ratio grows, and every result stays finite
    down to 2^-149."""
    figures = {e: pe.binade_ratio(e) for e in BINADES}
    print('\n' + '  '.join(f'2^{e}: {r:.2e}' for e, r in figures.items()))
    for e, r in figures.items():
        assert np.isfinite(r), e
        if e >= pe.CAP_FLOOR + 1:
            assert r <= BAR, (e, r)
    assert figures[-130] > BAR and figures[-149] > figures[-126] > figures[-120]     # the cap costs bits below 2^-108


def test_per_channel_results_are_finite_to_the_smallest_subnormal():
    """Channel maxima in every binade 2^-149 .. 2^100 against ReLU6 inputs and zero bias: every result is finite and
    no further from the float64 value than its S."""
    a = pe.relu6_rows(256, 96, 5)
    rng = np.random.default_rng(6)
    w = rng.uniform(-1.0, 1.0, (96, 250)) * np.ldexp(1.0, np.arange(-149, 101))[None, :]
    w[0] = 1.5 * np.ldexp(1.0, np.arange(-149, 101))
    w32 = pe.f32(w)
    got = pe.per_channel(a, w32, np.zeros(250, np.float32))
    assert np.isfinite(got).all()
    r = pe.ratios(got, a, w, np.zeros(250))
    assert (r <= 1.0).all(), float(r.max())
