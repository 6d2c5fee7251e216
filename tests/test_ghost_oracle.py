"""The GhostNet float64 oracle, the parameter container and the conv plan of the C ABI, on the CPU.

The oracle (oracle/ghost64.py) is what the GPU stages are held to, so it is checked first against the reference module
itself: the golden out102 of tests/golden/ref_vectors_ghostnet.npz was recorded from ghostnet_backbone.py on the CPU.
"""
import ctypes as C
import os
import types
from unittest import mock

import numpy as np
import pytest
import torch

from oracle import gemm64, ghost64, synth_ghost
from oracle import reference_port as rp
from synergynet_b200 import _lib, backbone, synthetic

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ref_vectors_ghostnet.npz')


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN, allow_pickle=False))


def golden_crops():
    return synthetic.normalize_crops(synthetic.make_structured_crops_u8(4, seed=31))


def test_float64_chain_matches_reference(gold):
    sd = synth_ghost.build_ghostnet_state_dict(0)
    out, feat = ghost64.forward64(sd, golden_crops())
    err = rp.max_rel_err(out.numpy(), gold['ghostnet_out102'])
    print(f'\n[ghostnet] float64 chain vs reference out102: {err:.3e}')
    assert err < 2e-5
    assert feat.shape == (4, 1280) and float(feat.min()) >= 0.0
    assert float(torch.from_numpy(gold['ghostnet_out102']).std(dim=0).min()) > 1e-3     # the faces differ


def test_params_keys_equal_reference_keys(gold):
    keys = list(backbone.ghostnet().state_dict().keys())
    assert keys == [str(k) for k in gold['ghostnet_keys']]


def test_conv_keys_follow_the_state_dict():
    sd = backbone.ghostnet().state_dict()
    keys = backbone.ghostnet_conv_keys()
    assert len(keys) == 95
    assert [c for c, _ in keys] == [k[:-len('.weight')] for k, v in sd.items() if k.endswith('.weight') and v.dim() == 4]
    for ck, bk in keys:
        assert (bk is None) == (ck + '.bias' in sd), ck
        if bk is not None:
            assert bk + '.running_var' in sd


def test_conv_plan_of_the_library_equals_the_module():
    lib = _lib.load()
    assert lib.syn_ghost_num_convs() == 95
    sd = backbone.ghostnet().state_dict()
    for i, (ck, _) in enumerate(backbone.ghostnet_conv_keys()):
        d = _lib.ConvDesc()
        _lib.check(lib.syn_ghost_conv_desc(i, C.byref(d)))
        w = sd[ck + '.weight']
        assert (d.cout, d.cin // d.groups, d.ksize, d.ksize) == tuple(w.shape), (i, ck)
        assert d.residual == int(ck.endswith('ghost2.cheap_operation.0')), ck
    for idx in (-1, 95):
        assert lib.syn_ghost_conv_desc(idx, C.byref(d)) == 1
    assert lib.syn_ghost_conv_desc(0, None) == 1


def test_stage_plan_of_the_library_equals_the_oracle():
    lib = _lib.load()
    table = ghost64.stage_table()
    assert lib.syn_ghost_num_stages() == len(table) == ghost64.NUM_STAGES == 111
    r, c, m = C.c_int(), C.c_int(), C.c_int()
    for s, st in enumerate(table):
        _lib.check(lib.syn_ghost_stage_desc(s, C.byref(r), C.byref(c), C.byref(m)))
        assert (r.value, c.value, bool(m.value)) == (st['rows'], st['cols'], st['rowmax']), (s, st['op'])
    assert lib.syn_ghost_stage_desc(len(table), C.byref(r), C.byref(c), C.byref(m)) == 1
    assert [b['ho'] for b in ghost64.blocks() if b['s'] > 1] == [30, 15, 8, 4]
    assert [i for i, b in enumerate(ghost64.blocks()) if b['red']] == [3, 4, 9, 10, 11, 13, 15]
    assert [i for i, b in enumerate(ghost64.blocks()) if b['short']] == [1, 3, 5, 9, 11]
    assert [b['red'] for b in ghost64.blocks() if b['red']] == [20, 32, 120, 168, 168, 240, 240]


def test_null_handle_calls_fail_cleanly():
    lib = _lib.load()
    assert lib.syn_ghost_set_conv_bias(None, 0, None, 0, None) == 1
    assert lib.syn_ghost_forward(None, None, 0, 1, None, None, None) == 1
    assert lib.syn_ghost_commit(None) == 1


def test_batches_cover_every_tile_shape():
    ghost64.check_ghost_batches()


@pytest.mark.parametrize('drop', [(33,), (128,), (129,), (2, 33, 128, 129)])
def test_each_batch_claim_fails_without_its_batches(drop):
    kept = tuple(b for b in ghost64.BATCHES if b not in drop)
    with pytest.raises(AssertionError):
        ghost64.check_ghost_batches(kept)


def test_faces_include_tile_edges():
    for b in ghost64.BATCHES:
        f = ghost64.faces(b)
        assert f[0] == 0 and f[-1] == b - 1 and f == sorted(set(f))


def test_reparametrisation_is_exact():
    """The rescaled checkpoint computes the same function: out102 of the float64 chain agrees to float64 rounding, while
    the hidden channels' magnitudes spread over 2^-6 .. 2^4."""
    sd = synth_ghost.build_ghostnet_state_dict(0)
    wide = synth_ghost.reparametrize_ghostnet(sd, seed=11, lo=-6, hi=4)
    x = golden_crops()[:2]
    a, _ = ghost64.forward64(sd, x)
    b, _ = ghost64.forward64(wide, x)
    assert rp.max_rel_err(b.numpy(), a.numpy()) < 1e-9
    g = wide['blocks.6.0.ghost1.cheap_operation.1.weight'] / sd['blocks.6.0.ghost1.cheap_operation.1.weight']
    assert float(g.min()) == 2.0 ** -6 and float(g.max()) == 2.0 ** 4


def test_gate_logits_reach_both_clamps():
    """On the golden crops, every SE block's conv_expand output lies below -3 and above +3 somewhere, so both clamps of
    relu6(z + 3) / 6 are exercised; its biases are non-zero."""
    sd = synth_ghost.build_ghostnet_state_dict(0)
    outs = {-1: golden_crops().double()}
    for s, st in enumerate(ghost64.stage_table()):
        outs[s] = ghost64.stage(sd, s, outs, 4)[0]
        if st['op'] == 'se_expand':
            z = outs[s]
            assert float(z.min()) < -3 and float(z.max()) > 3, st['block']
            p = ghost64.blocks()[st['block']]['p']
            assert bool((sd[p + 'se.conv_reduce.bias'] != 0).all() and (sd[p + 'se.conv_expand.bias'] != 0).all())


def test_se_padding_is_exact_in_float64():
    """The zero rows and columns the library adds to block 3's SE (20 -> 24 channels) change nothing: the padded reduce
    columns are exactly 0 and the expand output equals the unpadded one bit for bit."""
    sd = synth_ghost.build_ghostnet_state_dict(0)
    b = ghost64.blocks()[3]
    assert b['red'] == 20
    wr, br, we, be = ghost64.se_weights(sd, b)
    assert wr.shape == (24, 72) and we.shape == (72, 24)
    q = torch.randn(5, 72, dtype=torch.float64)
    z1 = (q @ wr.T + br).clamp_min(0.0)
    assert bool((z1[:, 20:] == 0).all())
    p = b['p'] + 'se.'
    w0r, w0e = sd[p + 'conv_reduce.weight'].double().reshape(20, 72), sd[p + 'conv_expand.weight'].double().reshape(72, 20)
    z1u = (q @ w0r.T + sd[p + 'conv_reduce.bias'].double()).clamp_min(0.0)
    assert torch.equal(z1[:, :20], z1u)
    assert torch.equal(z1 @ we.T + be, z1u @ w0e.T + sd[p + 'conv_expand.bias'].double())
    y, s = gemm64.gemm(q.float(), wr, br, True)
    assert bool((y[:, 20:] == 0).all() and (s[:, 20:] == 0).all())


def test_refusals_come_before_any_cuda_call():
    with mock.patch('torch.cuda.is_available', side_effect=AssertionError('CUDA touched')), \
            mock.patch('synergynet_b200._lib.load', side_effect=AssertionError('library touched')):
        for w in (0.5, 1.3, 2.0):
            with pytest.raises(RuntimeError, match='width 1.0'):
                backbone.ghostnet(width=w)
        m = backbone.ghostnet()
        with pytest.raises(RuntimeError, match='eval'):
            m(torch.zeros(1, 3, 120, 120))
        m.eval()
        for shape in ((1, 3, 112, 112), (1, 1, 120, 120), (3, 120, 120)):
            with pytest.raises(RuntimeError, match='120'):
                m(torch.zeros(shape))


def test_i2p_still_refuses_ghostnet():
    from synergynet_b200.model_building import I2P
    with pytest.raises(RuntimeError, match='mobilenet_v2 and resnet50 are built'):
        I2P(types.SimpleNamespace(arch='ghostnet'))
