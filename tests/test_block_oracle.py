"""CPU checks of the float64 per-stage oracle, its batch chooser and the wide-range checkpoint used by
tests/test_gpu_blocks.py."""
import pytest
import torch

from oracle import block64, synth_model, tile_cover
from oracle import reference_port as rp
from oracle.stage_check import LAYER_TOL, TAU, WIDE
from synergynet_b200 import _lib, synthetic
from synergynet_b200.backbone import conv_plan

PLAN = conv_plan()


@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def x8():
    from golden.vectors import load_ref_vectors
    return synthetic.normalize_crops(torch.from_numpy(load_ref_vectors()['x_u8']))


@pytest.fixture(scope='module')
def convs(sd, x8):
    """The fp32 oracle's 52 conv outputs of two faces, NHWC."""
    _, _, c = rp.mobilenetv2_forward(sd, x8[:2], return_convs=True)
    return [t.permute(0, 2, 3, 1).contiguous() for t in c]


def test_oracle_agrees_with_fp32_reference_per_conv_and_per_block(sd, x8, convs):
    """The float64 restatement computes what reference_port computes: the fp32 CPU convolutions (another summation
    order) sit under the bars the GPU engines are held to, per conv, per block and at the tail."""
    img = x8[:2]
    for spec in PLAN:
        src = img if spec.index == 0 else convs[spec.index - 1]
        skip = convs[spec.index - 3] if spec.residual else None
        r, where = block64.worst(convs[spec.index], *block64.conv(sd, spec.index, src, skip))
        assert r < TAU['tc_bf16x3']['conv'], (spec.index, r, where)
    for b in range(1, 18):
        src = img if b == 1 else convs[3 * b - 4]
        r, where = block64.worst(convs[3 * b - 1], *block64.block(sd, b, src))
        assert r < TAU['tc_fused']['block'], (b, r, where)
    pool, s = block64.tail(sd, convs[50])
    _, pool_ref = rp.mobilenetv2_forward(sd, img)
    assert block64.worst(pool_ref, pool, s)[0] < TAU['tc_fused']['pool']


def test_checker_flags_a_small_channel_that_max_rel_err_misses(sd, x8):
    """A channel whose values are a few percent of the tensor's maximum (a block output of the rescaled checkpoint),
    scaled by 1 + 1e-3: the per-element check flags it, while max_rel_err under the per-layer bar of test_gpu_parity
    passes the same tensor."""
    wide = synth_model.reparametrize_streams(sd, **WIDE['block64'])
    _, _, c = rp.mobilenetv2_forward(wide, x8[:2], return_convs=True)
    b = 9
    want, s = block64.block(wide, b, c[3 * b - 4].permute(0, 2, 3, 1))
    peak = want.abs().amax(dim=(0, 1, 2))
    small = ((peak > 0.01 * peak.max()) & (peak < 0.1 * peak.max())).nonzero().flatten()
    assert len(small) > 0
    c = int(small[0])
    bad = want.clone()
    bad[..., c] *= 1 + 1e-3
    assert rp.max_rel_err(bad.numpy(), want.numpy()) < LAYER_TOL[_lib.ENGINE_TC_FUSED]
    r, where = block64.worst(bad, want, s)
    assert r > 10 * TAU['tc_fused']['block'] and where[3] == c, (r, where)
    assert block64.worst(want.float(), want, s)[0] < TAU['tc_fused']['block']


def test_rescaled_checkpoint_is_exact_and_wide(sd, x8):
    """reparametrize_streams computes bit for bit the same params in fp32; every block input spreads its per-channel
    maxima over at least 2^8 and stays far inside the fp16 range of the split engines (|x| < ~937)."""
    wide = synth_model.reparametrize_streams(sd, **WIDE['block64'])
    p0, _, c0 = rp.mobilenetv2_forward(sd, x8, return_convs=True)
    p1, _, c1 = rp.mobilenetv2_forward(wide, x8, return_convs=True)
    assert torch.equal(p0, p1)
    block_inputs = [s.index - 1 for s in PLAN if s.kind in ('expand', 'last')]
    assert len(block_inputs) == 17
    for i in block_inputs:
        peak = c1[i].abs().amax(dim=(0, 2, 3)).double()
        assert peak.max() / peak.min() >= 2 ** 8, (i, float(peak.max() / peak.min()))
        assert peak.max() < 400, (i, float(peak.max()))
        f = peak / c0[i].abs().amax(dim=(0, 2, 3)).double()
        assert torch.equal(f, torch.exp2(torch.round(torch.log2(f)))), i          # exactly a power of two per channel


@pytest.mark.parametrize('sms', [114, 132])
def test_batch_chooser_covers_every_tile_plan(sms):
    batches = tile_cover.choose_batches(sms)
    for kind, batch in batches.items():
        tile_cover.check_plan(kind, batch, sms)
    # the numbers the plans come to on an H100 SXM (132 SMs) and PCIe (114 SMs)
    expect = {132: {'mixed_pairs': (330, 132, 198), 'odd_pairs': (199, 99, 100), 'ragged_quads': (531, 0, 133)},
              114: {'mixed_pairs': (284, 114, 170), 'odd_pairs': (171, 85, 86), 'ragged_quads': (459, 0, 115)}}[sms]
    for kind, (batch, split, groups) in expect.items():
        assert batches[kind] == batch
        assert tile_cover.tile_plan(batch, sms, 4 if kind == 'ragged_quads' else 2) == (split, groups)
    assert tile_cover.tail_ctas_per_slice(batches['odd_pairs'], sms) == sms // 10
    faces = tile_cover.faces_to_check(batches['mixed_pairs'], sms)
    assert {0, 2 * sms - 2, 2 * sms - 1, 2 * sms, batches['mixed_pairs'] - 1} <= set(faces)
    faces = tile_cover.faces_to_check(batches['ragged_quads'], sms)
    assert set(range(4 * sms, 4 * sms + 3)) <= set(faces) and len(faces) < 30


@pytest.mark.parametrize('sms', [114, 132])
def test_pool_placement_reaches_every_slot_and_tile_kind(sms):
    """The placement of tests/test_gpu_every_face.py: a 64-face pool over B = 1024 and the three tile-cover batches.
    Together the batches meet every claim; each batch drops only the claims its plans cannot meet."""
    pool = 64
    place = tile_cover.placement(1024, pool)
    assert place[:pool].tolist() == list(range(pool)) and place[pool:2 * pool].tolist() == list(range(1, pool)) + [0]
    assert torch.bincount(place).tolist() == [1024 // pool] * pool
    batches = {'bench': 1024, **tile_cover.choose_batches(sms)}
    met = {kind: tile_cover.check_placement(b, sms, pool) for kind, b in batches.items()}
    claims = set(met['bench'][0]) | set(met['bench'][1])
    assert len(claims) == 14
    for kind, (ok, dropped) in met.items():
        assert set(ok) | set(dropped) == claims and not set(ok) & set(dropped), kind
        assert all(dropped.values()), kind
    assert set().union(*(ok for ok, _ in met.values())) == claims
    # every pool face sits in both slots of the two-face groups, every slot of the four-face groups and of the tail
    # kernel's tiles, and at several row offsets of every map size, at B = 1024
    full = list(range(pool))
    bench = met['bench'][0]
    for claim in ['pair_both_slots', 'quad_every_slot', 'tail_every_slot'] + [f'rows{px}' for px in tile_cover.MAP_PIXELS]:
        assert bench[claim] == full, claim
    # what each plan cannot hold, on an H100 SXM (132 SMs) and PCIe (114 SMs)
    expect = {132: {'bench': {'single_face_group', 'quad_ragged_last'},
                    'mixed_pairs': {'tail_every_slot', 'later_tile_quad'},
                    'odd_pairs': {'tail_every_slot', 'later_tile_pair', 'later_tile_quad'},
                    'ragged_quads': set()},
              114: {'bench': {'quad_ragged_last'},
                    'mixed_pairs': {'quad_ragged_last', 'tail_every_slot', 'later_tile_quad'},
                    'odd_pairs': {'quad_every_slot', 'tail_every_slot', 'later_tile_pair', 'later_tile_quad'},
                    'ragged_quads': set()}}[sms]
    assert {kind: set(d) for kind, (_, d) in met.items()} == expect
    assert met['ragged_quads'][0]['quad_ragged_last'] == sorted(place[4 * sms:4 * sms + 3].tolist())
    # a batch smaller than the pool reaches no slot twice
    ok, dropped = tile_cover.check_placement(33, sms, pool)
    assert {'pair_both_slots', 'quad_every_slot', 'tail_every_slot'} <= set(dropped)
