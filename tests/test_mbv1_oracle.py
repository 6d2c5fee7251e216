"""The MobileNetV1 float64 oracle, the parameter container and the conv plan of the C ABI, on the CPU.

The oracle (oracle/mbv1_64.py) is what the GPU stages are held to, so it is checked first against the reference module
itself: the golden out102 of tests/golden/ref_vectors_mbv1.npz was recorded from mobilenetv1_backbone.py on the CPU.
"""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from oracle import mbv1_64, synth_mbv1
from oracle import reference_port as rp
from synergynet_b200 import _lib, backbone, synthetic

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ref_vectors_mbv1.npz')
ARCHS = tuple(backbone.MBV1_WIDTHS)
CODES = {'mobilenet_2': 200, 'mobilenet_1': 100, 'mobilenet_075': 75, 'mobilenet_05': 50, 'mobilenet_025': 25}


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN, allow_pickle=False))


def golden_crops():
    return synthetic.normalize_crops(synthetic.make_structured_crops_u8(4, seed=31))


@pytest.mark.parametrize('arch', ARCHS)
def test_float64_chain_matches_reference(gold, arch):
    sd = synth_mbv1.build_mobilenet_v1_state_dict(0, arch)
    out, pooled = mbv1_64.forward64(sd, golden_crops())
    err = rp.max_rel_err(out.numpy(), gold[f'{arch}_out102'])
    print(f'\n[{arch}] float64 chain vs reference out102: {err:.3e}')
    assert err < 2e-5
    assert pooled.shape == (4, int(1024 * backbone.MBV1_WIDTHS[arch]))


@pytest.mark.parametrize('arch', ARCHS)
def test_params_keys_equal_reference_keys(gold, arch):
    keys = list(getattr(backbone, arch)().state_dict().keys())
    assert keys == [str(k) for k in gold[f'{arch}_keys']]


@pytest.mark.parametrize('arch', ARCHS)
def test_conv_plan_of_the_library_equals_the_oracle_table(arch):
    lib = _lib.load()
    assert lib.syn_mbv1_num_convs() == 27
    table = mbv1_64.stage_table(arch)
    assert len(table) == 27
    for i, row in enumerate(table):
        d = _lib.ConvDesc()
        _lib.check(lib.syn_mbv1_conv_desc(CODES[arch], i, C.byref(d)))
        assert (d.cin, d.cout, d.ksize, d.stride, d.groups, d.h_in, d.h_out) == row, (arch, i)
        assert d.relu6 == 0 and d.residual == 0
    assert [r[6] for r in table[1::2]] == [60, 30, 30, 15, 15, 8, 8, 8, 8, 8, 8, 4, 4]    # 15 -> 8 with padding 1
    assert all(r[0] % 8 == 0 and r[1] % 8 == 0 for r in table[1:])


def test_unknown_widths_and_indices_are_rejected():
    lib = _lib.load()
    d = _lib.ConvDesc()
    for code in (0, 1, 2, 75 + 1, 150, 250, -100):
        assert lib.syn_mbv1_conv_desc(code, 0, C.byref(d)) == 1, code
        assert b'unknown widen code' in lib.syn_last_error()
    for idx in (-1, 27):
        assert lib.syn_mbv1_conv_desc(100, idx, C.byref(d)) == 1
    assert lib.syn_mbv1_conv_desc(100, 0, None) == 1
    assert lib.syn_mbv1_set_widen(None, 100) == 1
    assert lib.syn_mbv1_forward(None, None, 0, 1, None, None, None) == 1


def test_batches_cover_every_tile_shape():
    mbv1_64.check_mbv1_batches()


@pytest.mark.parametrize('drop, claim', [((33,), 'fewest rows'), ((128,), 'full tile'), ((2,), 'rows in between'),
                                         ((2, 33, 128), 'last partial band')])
def test_each_batch_claim_fails_without_its_batches(drop, claim):
    kept = tuple(b for b in mbv1_64.BATCHES if b not in drop)
    with pytest.raises(AssertionError):
        mbv1_64.check_mbv1_batches(kept)


def test_faces_include_tile_edges():
    for b in mbv1_64.BATCHES:
        f = mbv1_64.faces(b)
        assert f[0] == 0 and f[-1] == b - 1 and f == sorted(set(f))


@pytest.mark.parametrize('arch', ('mobilenet_1', 'mobilenet_025'))
def test_reparametrisation_is_exact(arch):
    """The rescaled checkpoint computes the same function: out102 of the float64 chain agrees to float64 rounding, while
    the hidden channels' magnitudes spread over 2^-6 .. 2^4."""
    sd = synth_mbv1.build_mobilenet_v1_state_dict(0, arch)
    wide = synth_mbv1.reparametrize_mobilenet_v1(sd, seed=11, lo=-6, hi=4)
    x = golden_crops()[:2]
    a, _ = mbv1_64.forward64(sd, x)
    b, _ = mbv1_64.forward64(wide, x)
    assert rp.max_rel_err(b.numpy(), a.numpy()) < 1e-9
    g = wide['dw3_1.bn_dw.weight'] / sd['dw3_1.bn_dw.weight']
    assert float(g.min()) == 2.0 ** -6 and float(g.max()) == 2.0 ** 4


def test_i2p_dispatch_of_mobilenet_names():
    from synergynet_b200.model_building import I2P
    for arch in ARCHS:
        m = I2P(types.SimpleNamespace(arch=arch))
        assert isinstance(m.backbone, backbone.MobileNetV1Params) and m._is_mbv1 and m._adapted
        assert m.backbone.widen_code == CODES[arch]
    with pytest.raises(RuntimeError, match='mobilenet_2, mobilenet_1, mobilenet_075, mobilenet_05, mobilenet_025'):
        I2P(types.SimpleNamespace(arch='mobilenet_3'))
    assert not I2P(types.SimpleNamespace(arch='mobilenet_v2'))._adapted
    for arch in ('ghostnet', 'resnest'):
        with pytest.raises(RuntimeError, match='mobilenet_v2 and resnet50 are built'):
            I2P(types.SimpleNamespace(arch=arch))
