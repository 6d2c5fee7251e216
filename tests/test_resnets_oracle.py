"""The ResNet float64 oracle, the parameter containers and the conv plans of the C ABI for the seven ResNet factories, on
the CPU.

The oracle (oracle/resnets64.py) is what the GPU stages are held to, so it is checked first against the reference modules
themselves: the golden out102 of tests/golden/ref_vectors_resnets.npz was recorded from resnet_backbone.py on the CPU.
"""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from oracle import gemm64, resnets64, synth_model, synth_resnet
from oracle import reference_port as rp
from synergynet_b200 import _lib, backbone, synthetic

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'ref_vectors_resnets.npz')
ARCHS = tuple(backbone.RESNET_ARCHS)
NEW = tuple(a for a in ARCHS if a != 'resnet50')
PREFIX = 'I2P.backbone.'


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLDEN, allow_pickle=False))


def golden_crops():
    return synthetic.normalize_crops(synthetic.make_structured_crops_u8(4, seed=31))


def prefixed(sd):
    return {PREFIX + k: v for k, v in sd.items()}


@pytest.mark.parametrize('arch', NEW)
def test_float64_chain_matches_reference(gold, arch):
    sd = prefixed(synth_resnet.build_resnet_state_dict(0, arch))
    out, pooled = resnets64.forward64(sd, golden_crops(), arch)
    err = rp.max_rel_err(out.numpy(), gold[f'{arch}_out102'])
    print(f'\n[{arch}] float64 chain vs reference out102: {err:.3e}')
    assert err < 2e-5
    assert pooled.shape == (4, 512 if backbone.RESNET_ARCHS[arch][0] < 50 else 2048)
    fp32, _ = resnets64.resnet_forward(sd, golden_crops(), arch)
    assert rp.max_rel_err(fp32.numpy(), gold[f'{arch}_out102']) < 2e-5


@pytest.mark.parametrize('arch', NEW)
def test_params_keys_equal_reference_keys(gold, arch):
    keys = list(getattr(backbone, arch)(pretrained=False).state_dict().keys())
    assert keys == [str(k) for k in gold[f'{arch}_keys']]
    assert list(synth_resnet.build_resnet_state_dict(0, arch)) == keys


@pytest.mark.parametrize('arch', ARCHS)
def test_conv_plan_of_the_library_equals_the_oracle_table(arch):
    lib = _lib.load()
    depth, wpg = backbone.RESNET_ARCHS[arch]
    table = resnets64.stage_table(arch)
    assert lib.syn_resnet_arch_num_convs(depth, wpg) == len(table) == len(backbone.resnet_conv_keys(arch))
    for i, row in enumerate(table):
        d = _lib.ConvDesc()
        _lib.check(lib.syn_resnet_arch_conv_desc(depth, wpg, i, C.byref(d)))
        assert (d.cin, d.cout, d.ksize, d.stride, d.h_in, d.h_out, bool(d.residual)) == row, (arch, i)
        assert d.groups == 1 and d.relu6 == 0
    assert all(r[0] % 8 == 0 and r[1] % 8 == 0 for r in table[1:])
    assert sorted({r[5] * r[5] for r in table[1:]}, reverse=True) == list(gemm64.RESNET_MAPS)
    n_res = sum(r[6] for r in table)
    assert n_res == len(resnets64.blocks(arch)) == sum(backbone.RESNET_LAYERS[depth])


def test_resnet50_table_equals_the_resnet50_entry_points():
    lib = _lib.load()
    assert lib.syn_resnet_num_convs() == lib.syn_resnet_arch_num_convs(50, 64) == 53
    for i in range(53):
        a, b = _lib.ConvDesc(), _lib.ConvDesc()
        _lib.check(lib.syn_resnet_conv_desc(i, C.byref(a)))
        _lib.check(lib.syn_resnet_arch_conv_desc(50, 64, i, C.byref(b)))
        assert bytes(a) == bytes(b), i
    assert backbone.resnet50_conv_keys() == backbone.resnet_conv_keys('resnet50')


def test_layer_table_of_the_issue():
    """Convs, max K and feature dim of every arch (the GMAC column of the docs follows from the same table)."""
    want = {'resnet18': (20, 4608, 512), 'resnet34': (36, 4608, 512), 'resnet50': (53, 4608, 2048),
            'resnet101': (104, 4608, 2048), 'resnet152': (155, 4608, 2048), 'wide_resnet50_2': (53, 9216, 2048),
            'wide_resnet101_2': (104, 9216, 2048)}
    for arch, (n, kmax, feat) in want.items():
        t = resnets64.stage_table(arch)
        assert (len(t), max(r[0] * r[2] ** 2 for r in t[1:]), t[-1][1]) == (n, kmax, feat), arch


def test_invalid_archs_and_indices_are_rejected():
    lib = _lib.load()
    d = _lib.ConvDesc()
    for depth, wpg in ((18, 128), (34, 128), (152, 128), (200, 64), (0, 64), (50, 32), (50, 0), (101, 256), (-50, 64)):
        assert lib.syn_resnet_arch_num_convs(depth, wpg) == -1, (depth, wpg)
        assert lib.syn_resnet_arch_conv_desc(depth, wpg, 0, C.byref(d)) == 1, (depth, wpg)
        msg = lib.syn_last_error()
        assert b'(18, 64)' in msg and b'(101, 128)' in msg, msg
        assert lib.syn_resnet_select(None, depth, wpg) == 1
    for depth, wpg in backbone.RESNET_ARCHS.values():
        n = lib.syn_resnet_arch_num_convs(depth, wpg)
        for idx in (-1, n):
            assert lib.syn_resnet_arch_conv_desc(depth, wpg, idx, C.byref(d)) == 1
        assert lib.syn_resnet_arch_conv_desc(depth, wpg, 0, None) == 1
    assert lib.syn_resnet_forward(None, None, 0, 1, None, None, None) == 1
    with pytest.raises(RuntimeError, match='no ResNet'):
        backbone.ResNetParams(18, 128)


def test_i2p_dispatch_of_resnet_names():
    from synergynet_b200.model_building import I2P
    for arch, (depth, wpg) in backbone.RESNET_ARCHS.items():
        m = I2P(types.SimpleNamespace(arch=arch))
        assert isinstance(m.backbone, backbone.ResNetParams) and m._is_resnet and m._adapted
        assert (m.backbone.depth, m.backbone.width_per_group) == (depth, wpg)
    listing = ', '.join(backbone.RESNET_ARCHS)
    for arch in ('resnet200', '_resnet', 'resnet50_2'):
        with pytest.raises(RuntimeError, match=listing):
            I2P(types.SimpleNamespace(arch=arch))
    for arch in ('ghostnet', 'resnest'):
        with pytest.raises(RuntimeError, match='mobilenet_v2 and resnet50 are built'):
            I2P(types.SimpleNamespace(arch=arch))
    for arch in ('vgg16', 'resnext50_32x4d'):
        with pytest.raises(RuntimeError, match='Please choose'):
            I2P(types.SimpleNamespace(arch=arch))


@pytest.mark.parametrize('arch', ('resnet18', 'wide_resnet50_2'))
def test_reparametrisation_is_exact(arch):
    """The rescaled checkpoint computes the same function: out102 of the float64 chain agrees to float64 rounding, while
    the hidden channels' magnitudes spread over 2^-6 .. 2^4."""
    sd = prefixed(synth_resnet.build_resnet_state_dict(0, arch))
    wide = synth_resnet.reparametrize_resnet(sd, arch, seed=11, lo=-6, hi=4, prefix=PREFIX)
    x = golden_crops()[:2]
    a, _ = resnets64.forward64(sd, x, arch)
    b, _ = resnets64.forward64(wide, x, arch)
    assert rp.max_rel_err(b.numpy(), a.numpy()) < 1e-9
    g = wide[PREFIX + 'layer2.1.bn1.weight'] / sd[PREFIX + 'layer2.1.bn1.weight']
    assert float(g.min()) == 2.0 ** -6 and float(g.max()) == 2.0 ** 4


def test_resnet50_checkpoint_and_oracle_are_those_of_the_resnet50_modules():
    """The generalised builders and oracle give ResNet-50 the bits its own builders and oracle give."""
    a, b = synth_model.build_resnet50_state_dict(0), synth_resnet.build_resnet_state_dict(0, 'resnet50')
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    wa = synth_model.reparametrize_resnet(a, seed=11, lo=-6, hi=4)
    wb = synth_resnet.reparametrize_resnet(b, 'resnet50', seed=11, lo=-6, hi=4)
    assert all(torch.equal(wa[k], wb[k]) for k in wa)
    sd = prefixed(a)
    x = golden_crops()[:2]
    o1, p1 = rp.resnet50_forward(sd, x)
    o2, p2 = resnets64.resnet_forward(sd, x)
    assert torch.equal(o1, o2) and torch.equal(p1, p2)
    stem = resnets64.stem(sd, x)
    assert all(torch.equal(u, v) for u, v in zip(stem, gemm64.resnet_stem(sd, x)))
    X = resnets64.maxpool(stem[0], 2).double()
    for i in (1, 2, 4):                                      # conv1, conv2 (3x3) and the downsample of layer1.0
        assert all(torch.equal(u, v) for u, v in zip(resnets64.conv(sd, i, X, 2), gemm64.resnet_conv(sd, i, X, 2)))
    pooled = torch.rand(2, 2048, dtype=torch.float64)
    assert all(torch.equal(u, v) for u, v in zip(resnets64.heads(sd, pooled), gemm64.resnet_heads(sd, pooled)))


def test_deep_checkpoints_stay_in_range():
    """The block-count scaling of the last BatchNorms keeps every arch's outputs at the magnitude of ResNet-50's."""
    x = golden_crops()
    for arch in ('resnet152', 'resnet101'):
        out, _ = resnets64.resnet_forward(prefixed(synth_resnet.build_resnet_state_dict(0, arch)), x, arch)
        assert 1.0 < float(out.abs().max()) < 1e3, arch
