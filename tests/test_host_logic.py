"""Host-side logic of the shim (no GPU): checkpoint schema, layer plan, index work, errors."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import reference_port as rp
from synergynet_b200 import _lib, inference, synthetic
from synergynet_b200.backbone import conv_plan


@pytest.fixture(scope='module')
def model(synth_pack):
    from synergynet_b200 import synergy3DMM
    return synergy3DMM.SynergyNet()


def test_state_dict_schema_matches_reference_counts(model):
    sd = model.state_dict()
    assert len(sd) == 445                                   # SURVEY.md section 8(b)
    assert sum(k.startswith('I2P.backbone.features.') for k in sd) == 312
    assert sum(k.startswith('forwardDirection.') for k in sd) == 63
    assert sum(k.startswith('reverseDirection.') for k in sd) == 56
    for name, shape in (('param_mean', (62,)), ('param_std', (62,)), ('w_shp', (159645, 40)),
                        ('u', (159645, 1)), ('w_exp', (159645, 10)), ('u_base', (204, 1)),
                        ('w_shp_base', (204, 40)), ('w_exp_base', (204, 10))):
        assert tuple(sd[name].shape) == shape
    assert tuple(sd['I2P.backbone.classifier_shape.1.weight'].shape) == (40, 1280)
    assert len(model.data_param) == 5 and model.data_param[3] is model.u_base


def test_conv_plan_covers_every_backbone_conv(model):
    plan = conv_plan()
    assert len(plan) == 52
    sd = model.state_dict()
    conv_keys = {k[:-len('.weight')] for k, v in sd.items()
                 if k.startswith('I2P.backbone.features.') and v.dim() == 4}
    assert {f'I2P.backbone.{s.conv_key}' for s in plan} == conv_keys
    for s in plan:
        w = sd[f'I2P.backbone.{s.conv_key}.weight']
        assert tuple(w.shape) == (s.cout, s.cin // s.groups, s.ksize, s.ksize)
        assert sd[f'I2P.backbone.{s.bn_key}.running_var'].shape[0] == s.cout
    macs = sum(s.h_out ** 2 * s.cout * (s.cin // s.groups) * s.ksize ** 2 for s in plan) + 62 * 1280
    assert macs == 93_204_560                                # SURVEY.md section 8(a)


def test_conv_plan_agrees_with_library():
    lib = _lib.load()
    assert lib.syn_num_conv_layers() == 52
    d = _lib.ConvDesc()
    for s in conv_plan():
        assert lib.syn_conv_desc(s.index, C.byref(d)) == 0
        assert (d.cin, d.cout, d.ksize, d.stride, d.groups, d.relu6, d.h_in, d.h_out, d.residual) == \
               (s.cin, s.cout, s.ksize, s.stride, s.groups, int(s.relu6), s.h_in, s.h_out, int(s.residual))
    assert lib.syn_conv_desc(52, C.byref(d)) == 1
    assert b'bad layer' in lib.syn_last_error()


def test_parse_param_62_bit_exact():
    from synergynet_b200.model_building import parse_param_62
    p = torch.randn(5, 62)
    got = parse_param_62(p)
    want = rp.parse_param_62(p.numpy())
    for g, w in zip(got, want):
        assert np.array_equal(g.numpy(), w)


def test_params_pack_gather_bit_exact(synth_pack):
    raw = synthetic.make_3dmm(0)
    want = rp.gather_sparse_basis(raw)
    for k in ('u', 'u_base', 'w_shp_base', 'w_exp_base'):
        assert np.array_equal(getattr(synth_pack, k), want[k])
    assert synth_pack.u_base.shape == (204, 1) and synth_pack.std_size == 120 and synth_pack.dim == 53215


def test_params_pack_missing_data(tmp_path):
    from synergynet_b200.params import ParamsPack
    with pytest.raises(RuntimeError, match='Missing data'):
        ParamsPack(data_dir=str(tmp_path))


def test_params_pack_reads_reference_file_layout(tmp_path):
    from synergynet_b200.params import ParamsPack
    raw = synthetic.make_3dmm(seed=4, nver=500)
    raw['tri'] = raw['tri'][:, :10] % 500 + 1
    synthetic.write_3dmm_dir(str(tmp_path), raw)
    pack = ParamsPack(data_dir=str(tmp_path))
    assert np.array_equal(pack.w_shp, raw['w_shp']) and np.array_equal(pack.keypoints, raw['keypoints'])
    assert np.array_equal(pack.u, raw['u_shp'] + raw['u_exp'])


def test_crop_img_matches_oracle_on_random_boxes():
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (83, 117, 3), dtype=np.uint8)
    for _ in range(200):
        x0, y0 = rng.uniform(-40, 100), rng.uniform(-40, 70)
        w, h = rng.uniform(1, 90), rng.uniform(1, 90)
        box = [x0, y0, x0 + w, y0 + h, 1.0]
        if x0 + w < 1 or y0 + h < 1 or x0 > 116 or y0 > 82:
            continue
        assert np.array_equal(inference.crop_img(img, box), rp.crop_img(img, box))
    gray = img[:, :, 0]
    assert np.array_equal(inference.crop_img(gray, [-3.2, 4.4, 50.5, 60.6, 1]), rp.crop_img(gray, [-3.2, 4.4, 50.5, 60.6, 1]))


def test_rescale_and_square_roi_match_oracle():
    v = np.random.default_rng(2).standard_normal((3, 68)).astype(np.float32) * 50
    box = [12.5, 7.25, 190.0, 201.5, 0.9]
    assert np.allclose(inference.rescale_vertices(v, box), rp.rescale_to_image(v, box), rtol=1e-6)
    sq = inference.square_roi([60.3, 80.1, 200.9, 250.4, 0.98])
    margin = (250.4 - 80.1) * 1.2 // 2
    assert sq[:4] == [(60.3 + 200.9) / 2 - margin, (80.1 + 250.4) / 2 - margin,
                      (60.3 + 200.9) / 2 + margin, (80.1 + 250.4) / 2 + margin] and sq[4] == 0.98


def test_reference_error_behaviour_without_gpu(model):
    with pytest.raises(RuntimeError, match='length of params mismatch'):
        model.reconstruct_vertex_62(torch.zeros(2, 61))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match='no CPU fallback'):
            model.forward_test(torch.zeros(1, 3, 120, 120))
    from synergynet_b200.model_building import I2P
    import types
    with pytest.raises(RuntimeError, match='Please choose'):
        I2P(types.SimpleNamespace(arch='vgg16'))


def test_product_package_never_imports_oracle():
    root = os.path.join(os.path.dirname(__file__), '..', 'synergynet_b200')
    for fn in os.listdir(root):
        if fn.endswith('.py'):
            src = open(os.path.join(root, fn)).read()
            assert 'import oracle' not in src and 'from oracle' not in src, fn


def test_shared_memory_lane_mappings_are_conflict_free():
    """Executable form of the layout claims in DESIGN.md section 5 (scripts/bank_check.py restates the kernel's
    lane -> address mappings): with the shipped choices every quarter-/half-warp access is conflict-free, and
    the rejected alternatives are exactly the 2-way conflicts ncu showed before the fixes."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location(
        'bank_check', os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'scripts', 'bank_check.py'))
    bc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bc)
    for name, (nc, w, s, ro) in bc.CONFIGS.items():
        assert bc.epi1_stores(nc) == 1, name
        assert bc.dw_octet_loads(nc, w, s, swap=(s == 2)) == 1, name            # quad swap only on stride 2
        assert bc.dw_octet_loads(nc, w, s, swap=(s != 2)) == 2, name
        if s == 1 and w in (8, 15, 30):                                         # register-blocked path
            assert bc.dw_quad_loads(nc, w, mirrored=True) == 1 and bc.dw_quad_loads(nc, w, mirrored=False) == 2, name
            assert bc.a2_quad_stores(w, mirrored=True) == 1 and bc.a2_quad_stores(w, mirrored=False) == 2, name


def test_render_module_has_the_reference_signature(synth_pack):
    """utils/render.py:31 -- same positional / keyword arguments and defaults; triangles come from the parameter pack."""
    import inspect
    from synergynet_b200 import render
    sig = inspect.signature(render.render)
    assert list(sig.parameters) == ['img', 'ver_lst', 'alpha', 'wfp', 'tex', 'connectivity']
    assert sig.parameters['alpha'].default == 0.6 and sig.parameters['wfp'].default is None
    assert render.cfg['intensity_ambient'] == 0.75 and render.cfg['specular_exp'] == 5          # utils/render.py:18-27
    assert callable(render.render_app) and hasattr(render.render_app, 'update_light_pos')
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match='no CPU fallback'):
            render.render(np.zeros((8, 8, 3), np.uint8), [np.zeros((3, synth_pack.tri.shape[1] and 53215), np.float32)])
