"""CPU checks of the float64 detector-network oracle (oracle/fb64.py), its stage table and its image-size chooser, used by
tests/test_gpu_fb_stages.py, and of the debug entry point's argument checks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import fb64
from oracle import render_port as rp
from synergynet_b200 import _lib, faceboxes, synthetic

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'render_vectors.npz')
TOL = 2e-5                  # max|a - b| / max|b|: the bar of the fp32 port in test_oracle_render.py


def _max_rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.fixture(scope='module')
def sd():
    return synthetic.make_faceboxes_state_dict(0)


@pytest.mark.parametrize('hw', [(250, 333, 0), (120, 96, 1)])
def test_oracle_chain_matches_reference_vectors(sd, hw):
    h, w, seed = hw
    gold = np.load(GOLD, allow_pickle=False)
    scene = synthetic.make_scene_u8(h, w, seed)
    outs, loc, conf = fb64.forward64(sd, torch.from_numpy(scene))
    l32, c32 = rp.faceboxes_forward(sd, scene)
    for got, want in ((loc, gold[f'fbs_loc_{h}x{w}']), (conf, gold[f'fbs_conf_{h}x{w}']), (loc, l32), (conf, c32)):
        assert got.shape == want.shape and _max_rel(got.numpy(), want) <= TOL
    for i in range(len(fb64.STAGES)):
        assert tuple(outs[i].shape) == faceboxes.debug_stage_shape(i, h, w), i


def test_stage_table_agrees_with_the_library():
    plan = faceboxes.layer_plan()
    assert len(plan) == len(fb64.LAYERS) == 33 and len(fb64.STAGES) == 39
    for L, p in zip(fb64.LAYERS, plan):
        assert (L.name, L.cin, L.cout, L.k, L.stride, L.pad, L.bn, L.act) == \
            (p['name'], p['cin'], p['cout'], p['ksize'], p['stride'], p['pad'], p['has_bn'], p['activation'])
    convs = [st.layer for st in fb64.STAGES if st.kind == 'conv']
    assert convs == list(range(33))                                     # every layer once, in execution order
    kinds = [st.kind for st in fb64.STAGES]
    assert kinds.count('maxpool') == 2 and kinds.count('avgpool') == 3 and kinds[-1] == 'softmax'
    for i, st in enumerate(fb64.STAGES):
        assert all(s == 'image' or s < i for s in st.inputs)
        if st.kind == 'conv' and st.dest not in ('loc', 'conf'):
            L = fb64.LAYERS[st.layer]
            assert st.owns[1] - st.owns[0] == L.cout * (2 if L.act == 2 else 1), i      # CReLU writes 2 x cout
        if st.kind == 'conv' and st.layer > 0:
            src = fb64.STAGES[st.inputs[0]]                               # reads a whole tensor of cin channels
            h, w = fb64.PRODUCTION
            assert faceboxes.debug_stage_shape(st.inputs[0], h, w)[2] == fb64.LAYERS[st.layer].cin, (i, src)
    # every inception block's four branches tile its 128 channels
    for last in fb64.BLOCK_LAST:
        owns = sorted(fb64.STAGES[s].owns for s in range(last - 7, last + 1) if fb64.STAGES[s].dest == fb64.STAGES[last].dest)
        assert owns == [(0, 32), (32, 64), (64, 96), (96, 128)]
    h, w = 250, 333
    assert fb64.head_range(34, h, w)[1] == 4 * fb64.num_priors(h, w) == 4 * rp.prior_boxes(h, w).shape[0]
    assert fb64.head_range(37, h, w)[1] == 2 * fb64.num_priors(h, w)


def test_size_chooser_covers_every_claim():
    sizes = fb64.choose_sizes()
    fb64.check_sizes(sizes)
    assert len(sizes) <= 10
    for name, ok in fb64.claims().items():                              # each claim holds only through the sizes it names
        rest = [s for s in sizes if not ok(*s)]
        assert len(rest) < len(sizes), name
        with pytest.raises(AssertionError, match=name):
            fb64.check_sizes(rest)
    # the sizes that pin a 64-row last tile on the stride-32 / -64 / -128 maps
    rows = lambda hw, m: fb64.maps(*hw)[m][0] * fb64.maps(*hw)[m][1]
    assert rows((33, 993), 's0') == 64 and rows((193, 961), 's1') == 64 and rows((1024, 1024), 's2') == 64


def test_debug_entry_rejects_bad_arguments_without_a_device():
    lib = _lib.load()
    buf = C.c_void_p(16)                                                  # never dereferenced: the checks come first
    for stage in (-1, 39):
        assert lib.syn_fb_debug_forward_until(None, buf, 64, 64, stage, buf, 1, buf, buf, None) == 1
        assert b'stage' in lib.syn_last_error()
    assert lib.syn_fb_debug_forward_until(None, buf, 64, 64, 0, buf, 1, buf, buf, None) == 1
    assert b'null handle' in lib.syn_last_error()
    with pytest.raises(ValueError):
        faceboxes.debug_stage_shape(39, 64, 64)
