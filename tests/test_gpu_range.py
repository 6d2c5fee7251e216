"""The edge of the split-fp16 engines' input range, against the float64 oracle (oracle/block64.py).  H100 only.

Engines 1-3 multiply an activation by kActScale = 64 and clamp it to +-60000 before the fp16 hi/lo split, so an input
|x| > 937.5 (or +-Inf, or NaN) is changed; the sticky flag ``poll_saturation`` must then be raised.  The clamp sits at
three places: the fused kernel's input conversion (the fp32 crop of the stem and the inputs of blocks 2-17, engines 2
and 3), the tail kernel's producers (the block-17 output, engines 2 and 3) and the A conversion of the tensor-core
pointwise conv (every expand and conv 51, engine 1).

One channel of a block stream is rescaled (``synth_model.scale_stream_channel``) so that its largest value over the
tile-cover batch, taken from the fp32 engine, becomes 0.995 or 1.005 x 937.5:

  inside    no flag on any engine, and every stage of engines 0-2 under the per-element bar of
            ``oracle/stage_check.py`` with hi/lo operands at the top of the fp16 range (all seven streams at once);
  outside   the flag on every engine that clamps the stream and not on engine 0, which still passes the bar; the stage
            that reads the stream passes the bar against the oracle fed clip(x, -937.5, 937.5) and fails it against
            the unclamped input, so the clamp sits exactly at 60000 / 64 and changes nothing else.

The crop itself is probed pixel by pixel at the stem strips' edge rows and columns, with 937.5, its fp32 successor,
+Inf and NaN.
"""
import math

import numpy as np
import pytest
import torch

from oracle import block64, stage_check, synth_model, tile_cover
from oracle.stage_check import make_model, report, seeded_crops, stage_ratios, tau
from synergynet_b200 import _lib

pytestmark = pytest.mark.gpu

LIMIT = 60000.0 / block64.ACT_SCALE                  # 937.5: the largest |x| the split engines take unchanged
INSIDE, OUTSIDE = 0.995 * LIMIT, 1.005 * LIMIT
NAMES = {v: k for k, v in stage_check.ENGINES.items()}
ALL = (_lib.ENGINE_SIMT_FP32, _lib.ENGINE_TC_BF16X3, _lib.ENGINE_TC_FUSED, _lib.ENGINE_TC_FUSED_1PASS)
# (channel, row, column) of the crop pixels probed: rows 9 and 25 are the first and last input rows of stem strip 1
# (hidden rows 5..12; strips 0 and 2 read them too), rows 0 and 119 those of the first and last strip, where the zero
# pad lies; columns 0 and 119 are the two padded edges of the im2col gather
PIXELS = ((0, 9, 0), (1, 25, 119), (2, 0, 119), (1, 119, 0))
CROP_BATCH, CROP_FACE = 6, 3


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


def _stream_peak(eng, x, stream, channel=None):
    """(channel, max |x|, face) of the stream over its block inputs (the outputs of the blocks that write it):
    the channel with the largest value, or the given one."""
    best = None
    for b in synth_model.stream_blocks(stream)[0]:
        y = eng.debug_forward_until(x, 3 * b - 1).abs()
        peak = y.amax(dim=(0, 1, 2))
        c = int(torch.argmax(peak)) if channel is None else channel
        if best is None or float(peak[c]) > best[1]:
            best = (c, float(peak[c]), int(y[..., c].amax(dim=(1, 2)).argmax()))
    return best


@pytest.fixture(scope='module')
def peaks(synth_pack, sd, batch):
    """{stream: (channel, max |x|, face)} of the fp32 engine on the tile-cover batch."""
    eng = _engine(make_model(sd), _lib.ENGINE_SIMT_FP32)
    return {s: _stream_peak(eng, batch[0], s) for s in synth_model.STREAMS}


def _scaled(sd, peaks, streams, target):
    for s in streams:
        c, m, _ = peaks[s]
        sd = synth_model.scale_stream_channel(sd, s, c, target / m)
    return sd


def _faces(batch, peaks, streams):
    return sorted(set(batch[1]) | {peaks[s][2] for s in streams})


def _run_flag(eng, x):
    eng.forward(x)
    assert eng.poll_error() == 0
    return eng.poll_saturation(warn=False)


@pytest.fixture(scope='module')
def inside(synth_pack, sd, peaks):
    sd_in = _scaled(sd, peaks, synth_model.STREAMS, INSIDE)
    return sd_in, make_model(sd_in)


def test_inside_the_range_raises_no_flag(inside, peaks, batch):
    sd_in, model = inside
    x = batch[0]
    try:
        eng = _engine(model, _lib.ENGINE_SIMT_FP32)
        for s in synth_model.STREAMS:
            c, m, _ = _stream_peak(eng, x, s, peaks[s][0])
            assert 0.99 * LIMIT < m <= LIMIT, (s, c, m)                  # the channel really sits at the top
        for kind in ALL:
            assert _run_flag(_engine(model, kind), x) == 0, kind
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)


@pytest.mark.parametrize('engine', list(stage_check.ENGINES))
def test_inside_the_range_every_stage_matches_float64_oracle(inside, peaks, batch, engine):
    sd_in, model = inside
    x, faces = batch[0], _faces(batch, peaks, synth_model.STREAMS)
    try:
        ratios = stage_ratios(_engine(model, stage_check.ENGINES[engine]), engine == 'tc_fused', sd_in, x, faces)
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)
    report(f'{engine} inside, every stream at {INSIDE / LIMIT:.3f} x 937.5, faces={len(faces)}', ratios)
    bad = stage_check.over(engine, ratios)
    assert not bad, bad


def _consumer_ratios(eng, fused, sd, x, faces, readers):
    """{stage reading the stream: (ratio against the oracle fed the clamped input, against the unclamped input)}.
    Engine 1 reads it in the expand conv of each reader block and in conv 51; the fused engine in the whole block (whose
    skip adds the unclamped fp32 input) and in the tail kernel (checked on the pooled feature)."""
    fidx = torch.tensor(faces, device='cuda')
    pick = lambda t: t.index_select(0, fidx).cpu().double()
    out = {}
    for b in readers:
        idx = 51 if b == 18 else 3 * b - 3                  # conv reading the stream; its input is conv idx - 1
        prev = pick(eng.debug_forward_until(x, idx - 1))
        clip = prev.clamp(-LIMIT, LIMIT)
        if not fused:
            got, name = pick(eng.debug_forward_until(x, idx)), f'conv{idx}'
            want = (block64.conv(sd, idx, clip), block64.conv(sd, idx, prev))
        elif b <= 17:
            got, name = pick(eng.debug_forward_until(x, 3 * b - 1)), f'block{b}'
            want = (block64.block(sd, b, clip, skip=prev), block64.block(sd, b, prev))
        else:
            got, name = pick(eng.forward(x, want_pool=True)[1]), 'pool'
            want = (block64.tail(sd, clip), block64.tail(sd, prev))
        out[name] = tuple(block64.worst(got, *w) for w in want)
    return out


@pytest.mark.parametrize('stream', synth_model.STREAMS)
def test_just_outside_the_range(synth_pack, sd, peaks, batch, stream):
    sd_out = _scaled(sd, peaks, [stream], OUTSIDE)
    model = make_model(sd_out)
    x, faces = batch[0], _faces(batch, peaks, [stream])
    readers = synth_model.stream_blocks(stream)[1]
    try:
        flags = {kind: _run_flag(_engine(model, kind), x) for kind in ALL}
        assert flags == {kind: int(kind != _lib.ENGINE_SIMT_FP32) for kind in ALL}, (stream, flags)
        eng = _engine(model, _lib.ENGINE_SIMT_FP32)
        c, m, _ = _stream_peak(eng, x, stream, peaks[stream][0])
        assert LIMIT < m < 1.01 * LIMIT, (stream, c, m)
        ratios = stage_ratios(eng, False, sd_out, x, faces)          # also: engine 0 raises no flag
        report(f'simt_fp32 outside, stream {stream} channel {c} at {m / LIMIT:.4f} x 937.5', ratios)
        bad = stage_check.over('simt_fp32', ratios)
        assert not bad, bad
        for engine in ('tc_bf16x3', 'tc_fused'):
            eng = _engine(model, stage_check.ENGINES[engine])
            got = _consumer_ratios(eng, engine == 'tc_fused', sd_out, x, faces, readers)
            assert eng.poll_saturation(warn=False) == 1
            print(f'[{engine} outside, stream {stream}] ' + '  '.join(
                f'{k}: clamped {v[0][0]:.2e} unclamped {v[1][0]:.2e}' for k, v in got.items()))
            bad = {k: v[0] for k, v in got.items() if v[0][0] > tau(engine, k)}
            assert not bad, bad
            assert any(v[1][0] > tau(engine, k) for k, v in got.items()), got
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)


def _crops():
    return seeded_crops(CROP_BATCH, 77)


def _with_pixel(x, pixel, value):
    x = x.clone()
    c, r, col = pixel
    x[CROP_FACE, c, r, col] = value
    return x


@pytest.fixture(scope='module')
def model(synth_pack, sd):
    return make_model(sd)


@pytest.mark.parametrize('kind', [_lib.ENGINE_TC_FUSED, _lib.ENGINE_TC_FUSED_1PASS])
def test_crop_pixels_at_the_edge_of_the_range(model, sd, kind):
    """A single crop pixel of the fused stem: +-937.5 passes unchanged and raises no flag; its fp32 successor, +Inf and
    NaN raise it.  The clamped face's block 1 is what the oracle gives for the clamped crop (NaN is read as -937.5)
    on the split-fp16x3 engine, and every other face of the batch is bit-identical to the same call with the pixel
    at 0."""
    eng = _engine(model, kind)
    x0 = _crops()
    above = float(np.nextafter(np.float32(LIMIT), np.float32(np.inf)))          # the fp32 successor of 937.5
    cases = ((LIMIT, 0, LIMIT), (-LIMIT, 0, -LIMIT), (above, 1, LIMIT), (math.inf, 1, LIMIT), (math.nan, 1, -LIMIT))
    others = [f for f in range(CROP_BATCH) if f != CROP_FACE]
    worst = 0.0
    try:
        for pixel in PIXELS:
            base = _with_pixel(x0, pixel, 0.0)
            ref_p, ref_b1 = eng.forward(base), eng.debug_forward_until(base, 2)
            assert _run_flag(eng, base) == 0
            for value, flag, clamped in cases:
                x = _with_pixel(x0, pixel, value)
                params, b1 = eng.forward(x), eng.debug_forward_until(x, 2)
                assert eng.poll_error() == 0
                assert eng.poll_saturation(warn=False) == flag, (pixel, value)
                assert torch.equal(params[others], ref_p[others]) and torch.equal(b1[others], ref_b1[others]), \
                    (pixel, value)
                assert bool(torch.isfinite(params).all()) and bool(torch.isfinite(b1).all())
                if kind == _lib.ENGINE_TC_FUSED:
                    img = _with_pixel(x0, pixel, clamped)[CROP_FACE:CROP_FACE + 1].cpu()
                    r, where = block64.worst(b1[CROP_FACE:CROP_FACE + 1].cpu(), *block64.block(sd, 1, img))
                    assert r <= tau('tc_fused', 'block'), (pixel, value, r, where)
                    worst = max(worst, r)
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)
    if kind == _lib.ENGINE_TC_FUSED:
        print(f'\n[tc_fused crop pixels] worst block-1 ratio {worst:.3e}')


@pytest.mark.parametrize('kind', [_lib.ENGINE_SIMT_FP32, _lib.ENGINE_TC_BF16X3])
def test_fp32_stem_takes_pixels_beyond_the_range(model, sd, kind):
    """Engines 0 and 1 run the stem in fp32 and clamp nothing there: at 4 x 937.5 no flag, and the stem and block 1
    (convs 0-2) stay under the bar."""
    eng = _engine(model, kind)
    name = NAMES[kind]
    x = _crops()
    for pixel in PIXELS:
        x = _with_pixel(x, pixel, 4 * LIMIT if pixel[2] == 0 else -4 * LIMIT)
    face = slice(CROP_FACE, CROP_FACE + 1)
    try:
        prev = x[face].cpu()
        for i in range(3):
            got = eng.debug_forward_until(x, i)[face].cpu()
            r, where = block64.worst(got, *block64.conv(sd, i, prev))
            assert r <= tau(name, 'conv'), (i, r, where)
            prev = got
        assert _run_flag(eng, x) == 0
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)


def test_flag_is_sticky_cleared_by_the_poll_and_per_handle(synth_pack, sd, model):
    """A NaN crop raises the flag of its handle; later clean calls keep it; the poll reports and clears it; a second
    model on the same device never sees it."""
    other = make_model(sd)
    eng, eng2 = _engine(model, _lib.ENGINE_TC_FUSED), _engine(other, _lib.ENGINE_TC_FUSED)
    assert eng is not eng2
    x = _crops()
    assert eng.poll_saturation(warn=False) == 0 and eng2.poll_saturation(warn=False) == 0
    eng.forward(_with_pixel(x, PIXELS[0], math.nan))
    eng2.forward(x)
    eng.forward(x)
    eng.forward(x)
    assert eng2.poll_saturation(warn=False) == 0
    assert eng.poll_saturation(warn=False) == 1
    assert eng.poll_saturation(warn=False) == 0
    eng.forward(x)
    assert eng.poll_saturation(warn=False) == 0
