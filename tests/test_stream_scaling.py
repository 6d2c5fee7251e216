"""CPU checks of ``synth_model.scale_stream_channel``, the checkpoint edit that puts one channel of a block stream at
the edge of the split-fp16 engines' range for tests/test_gpu_range.py."""
import pytest
import torch

from oracle import block64, synth_model
from synergynet_b200.backbone import conv_plan

REL = 1e-6


@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def x3():
    from golden.vectors import load_ref_vectors
    from synergynet_b200 import synthetic
    return synthetic.normalize_crops(torch.from_numpy(load_ref_vectors()['x_u8'][:3]))


def _chain(sd, x):
    """Float64 block outputs 1..17 of the oracle, then the pooled feature and the params."""
    outs, prev = [], x
    for b in range(1, 18):
        prev = block64.block(sd, b, prev)[0]
        outs.append(prev)
    pool = block64.tail(sd, prev)[0]
    return outs, pool, block64.heads(sd, pool)[0]


@pytest.fixture(scope='module')
def base(sd, x3):
    return _chain(sd, x3)


def _close(got, want, scale):
    return float((got - want).abs().max()) <= REL * scale


def test_stream_table():
    got = {s: synth_model.stream_blocks(s) for s in synth_model.STREAMS}
    assert got == {16: ([1], [2]), 24: ([2, 3], [3, 4]), 32: ([4, 5, 6], [5, 6, 7]), 64: ([7, 8, 9, 10], [8, 9, 10, 11]),
                   96: ([11, 12, 13], [12, 13, 14]), 160: ([14, 15, 16], [15, 16, 17]), 320: ([17], [18])}


@pytest.mark.parametrize('stream', synth_model.STREAMS)
def test_moves_exactly_one_channel_of_one_stream(sd, x3, base, stream):
    """At every block input of the stream the chosen channel is ``factor`` times the original and every other channel
    is unchanged; every other block output, the pooled feature and the params are unchanged (float64 oracle, fp32
    weights, so to the rounding of the rescaled weights)."""
    channel, factor = stream // 3, 93.7
    outs, pool, params = _chain(synth_model.scale_stream_channel(sd, stream, channel, factor), x3)
    writers, _ = synth_model.stream_blocks(stream)
    for b in range(1, 18):
        got, want = outs[b - 1], base[0][b - 1]
        if b in writers:
            others = [c for c in range(want.shape[-1]) if c != channel]
            peak = float(want[..., channel].abs().max())
            assert peak > 0, (stream, b)
            assert _close(got[..., channel], factor * want[..., channel], factor * peak), (stream, b)
            assert _close(got[..., others], want[..., others], float(want.abs().max())), (stream, b)
            assert not _close(got[..., channel], want[..., channel], peak), (stream, b)
        else:
            assert _close(got, want, float(want.abs().max())), (stream, b)
    assert _close(pool, base[1], float(base[1].abs().max()))
    assert _close(params, base[2], float(base[2].abs().max()))


@pytest.mark.parametrize('stream', synth_model.STREAMS)
def test_power_of_two_factor_is_reparametrize_streams_arithmetic(sd, stream):
    """With the factor reparametrize_streams drew for a channel, the helper writes bit for bit the values
    reparametrize_streams wrote into that channel's BatchNorm entries and weight columns, and touches nothing else."""
    wide = synth_model.reparametrize_streams(sd, seed=7, lo=-6, hi=4)
    pre = 'I2P.backbone.'
    writers = [s for s in conv_plan() if s.kind == 'project' and s.cout == stream]
    readers = [s for s in conv_plan() if s.kind in ('expand', 'last') and s.cin == stream]
    key = pre + writers[0].bn_key + '.weight'
    for channel in (0, stream - 1):
        factor = float(wide[key][channel] / sd[key][channel])
        assert factor == 2.0 ** round(torch.log2(torch.tensor(factor)).item()), factor
        got = synth_model.scale_stream_channel(sd, stream, channel, factor)
        want = {k: v.clone() for k, v in sd.items()}
        for s in writers:
            for k in ('.weight', '.bias'):
                want[pre + s.bn_key + k][channel] = wide[pre + s.bn_key + k][channel]
        for s in readers:
            want[pre + s.conv_key + '.weight'][:, channel] = wide[pre + s.conv_key + '.weight'][:, channel]
        assert got.keys() == sd.keys()
        assert all(torch.equal(got[k], want[k]) for k in sd), (stream, channel)
        assert sum(not torch.equal(got[k], sd[k]) for k in sd) == 2 * len(writers) + len(readers) or factor == 1.0
