"""The ResNet backbones other than ResNet-50 on the H100 (resnet18 / 34 / 101 / 152, wide_resnet50_2 / wide_resnet101_2):
every stage of every arch against the float64 oracle (oracle/resnets64.py), element by element, then end to end against
the reference modules' golden outputs and through the reference's caller sequences.  ResNet-50 itself is checked stage by
stage in test_gpu_gemm_layers.py; here its generic entry point is held to the ResNet-50 one bit for bit.

Each stage is fed the GPU's own output of the previous stage and held to |got - want| <= TAU * S; the max-pool and every
row maximum a stage records are compared bit for bit.  The batches put the last 128-row tile of every map size in each
of its shapes (gemm64.check_resnet_batches); the faces checked include the last face and the faces around the last
tile's edge (gemm64.resnet_faces).
"""
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import gemm64, resnets64, synth_resnet
from oracle.stage_check import TAU, WIDE, Ratios, check_rowmax, face_picker, make_model, report, same_bits, seeded_crops
from oracle import reference_port as rp
from synergynet_b200 import backbone, synthetic

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
ARCHS = tuple(a for a in backbone.RESNET_ARCHS if a != 'resnet50')
BARS = TAU['gemm64']
GOLD_FACES, GOLD_SEED = 4, 31             # tests/golden/make_golden_resnets.py
# End to end, out102 and the landmarks against the reference modules' fp32 outputs.  Every stage is held to its bar above;
# what reaches out102 is then set by the checkpoint's conditioning: the four heads sum 512 or 2048 non-negative pooled
# features with weights of both signs, so |out102| is ~40x below the sum of |a||w| the stage bar is relative to, and the
# reconstruction amplifies the parameters' error ~1.6x again.  On the float64 oracle, noise of 1e-6 x S injected at every
# conv moves out102 by 3.5e-5 for resnet50 and 3.2e-5 for wide_resnet50_2, and at the heads alone by 2.9e-5 / 4.0e-5.
# Measured on an H100 80GB HBM3 (700 W power limit): out102 6.2e-05 (resnet18) .. 1.48e-04 (wide_resnet101_2), landmarks
# 1.18e-04 (resnet18) .. 2.32e-04 (wide_resnet50_2); resnet50, built the same way, measures 9e-5 against its 1e-4.  The
# bar is 4e-4, under 2x the worst.
E2E_TOL = 4e-4


@pytest.fixture(scope='module')
def gold():
    import os
    return dict(np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_vectors_resnets.npz'), allow_pickle=False))


def checkpoint(arch, seed=0):
    return synth_resnet.build_resnet_state_dict(seed, arch)


@pytest.fixture(scope='module')
def models(synth_pack):
    return {}


def model_of(models, arch):
    if arch not in models:
        models[arch] = make_model(checkpoint(arch), arch, strict=False)
    return models[arch]


def kind_of(arch, i):
    """'gemm' for every GEMM conv; the K = 9216 convs of the wide arches are reported on their own as 'gemm9216', under
    the same bar (the GEMM ratio grows with K: they measure 3.79e-06 on an H100 80GB HBM3 at 700 W, against 2.58e-06 for
    the K = 4608 convs of these arches and the bar's 8e-6)."""
    cin, _, k, _, _, _, _ = resnets64.stage_table(arch)[i]
    return 'gemm9216' if cin * k * k > 4608 else 'gemm'


def bar(kind):
    return BARS['gemm' if kind.startswith('gemm') else kind]


def resnet_ratios(eng, sd, arch, x, faces, ratios):
    """Run every stage of ``arch`` on batch ``x`` and hold the given faces to the oracle; row maxima bit for bit."""
    nf = len(faces)
    keys = resnets64.conv_keys(arch)
    n = len(keys)
    pick, where = face_picker(x.shape[0], faces, x.device)

    def run(stage, name):
        out, rm = eng.debug_resnet_until(x, stage)
        if rm is not None:
            check_rowmax(out, rm, name)
        return pick(out)

    stem = run(0, 'stem')
    ratios.add('simt', 'stem', stem, resnets64.stem(sd, x[faces].cpu(), arch), where(3600))
    pool = run(1, 'maxpool')
    assert same_bits(pool, resnets64.maxpool(stem, nf)), 'maxpool'

    def conv(i, inp, residual=None):
        got = run(1 + i, keys[i][0])
        want = resnets64.conv(sd, i, inp, nf, residual, arch)
        ratios.add(kind_of(arch, i), keys[i][0], got, want, where(got.shape[0] // nf))
        return got

    X = pool
    for inner, last, ds in resnets64.blocks(arch):
        cur = X
        for i in inner:
            cur = conv(i, cur)
        ident = conv(ds, X) if ds is not None else X
        X = conv(last, cur, ident)
    pooled = run(n + 1, 'avgpool')
    ratios.add('pool', 'avgpool', pooled, resnets64.avgpool(X, nf), where(1))
    heads = run(n + 2, 'heads')
    ratios.add('gemm', 'heads', heads, resnets64.heads(sd, pooled), where(1))
    assert eng.poll_error() == 0


def above_bar(ratios):
    return {s: v for s, v in ratios.items() if v[0] > bar(v[2])}


@pytest.mark.parametrize('batch', resnets64.BATCHES)
@pytest.mark.parametrize('arch', ARCHS)
def test_every_stage_matches_float64_oracle(models, arch, batch):
    gemm64.check_resnet_batches()
    faces = resnets64.faces(batch)
    gemm64.check_resnet_faces(batch, faces)
    sd = {'I2P.backbone.' + k: v for k, v in checkpoint(arch).items()}
    eng = model_of(models, arch)._engine(DEV)
    ratios = Ratios()
    resnet_ratios(eng, sd, arch, seeded_crops(batch, 500 + batch), faces, ratios)
    report(f'{arch} B={batch} faces={faces}', ratios)
    bad = above_bar(ratios)
    assert not bad, bad


@pytest.mark.parametrize('arch', ARCHS)
def test_rescaled_checkpoint(synth_pack, gold, arch):
    """Hidden channels spread over 2^10: the same function (out102 of the reference within E2E_TOL) and every stage under
    the same bar, with the GEMMs' row scales spread as widely."""
    sd = synth_resnet.reparametrize_resnet(checkpoint(arch), arch, **WIDE['gemm64'])
    eng = make_model(sd, arch, strict=False)._engine(DEV)
    out, _ = eng.forward_resnet(seeded_crops(GOLD_FACES, GOLD_SEED))
    err = rp.max_rel_err(out.cpu().numpy(), gold[f'{arch}_out102'])
    print(f'\n[{arch} rescaled] out102 err {err:.3e}')
    assert err < E2E_TOL
    batch = resnets64.BATCHES[0]
    ratios = Ratios()
    resnet_ratios(eng, {'I2P.backbone.' + k: v for k, v in sd.items()}, arch, seeded_crops(batch, 500 + batch),
                  resnets64.faces(batch), ratios)
    report(f'{arch} rescaled B={batch}', ratios)
    bad = above_bar(ratios)
    assert not bad, bad


def test_negative_control_fails_the_bar(models):
    """A K = 9216 conv (wide_resnet50_2 layer4.1.conv2, 3x3 over 1024 channels) on the GPU's own conv1 output through the
    same GEMM: with the true weights it passes; with its weights rounded to bf16 it must fail by >= 10x."""
    arch, batch = 'wide_resnet50_2', 3
    keys = resnets64.conv_keys(arch)
    idx = [ck for ck, _ in keys].index('layer4.1.conv2')
    cin, _, k, s, hin, ho, _ = resnets64.stage_table(arch)[idx]
    assert cin * k * k == 9216
    sd = {'I2P.backbone.' + kk: v for kk, v in checkpoint(arch).items()}
    eng = model_of(models, arch)._engine(DEV)
    x = seeded_crops(batch, 5)
    a, rm = eng.debug_resnet_until(x, idx)                 # conv idx - 1 = layer4.1.conv1, the input of conv idx
    w, b = resnets64.fold(sd, idx, arch)
    w = w.float()
    want = resnets64.conv(sd, idx, a.cpu(), batch, None, arch)
    maps = a.view(batch, hin, hin, cin)
    ratio = lambda weights: gemm64.worst(eng.debug_gemm(weights, b.float(), maps, rm, act=2, conv=(k, s, 1, ho, ho))[0].cpu(),
                                         *want)[0]
    r_ok, r_bf16 = ratio(w), ratio(w.bfloat16().float())
    print(f'\n[negative control K=9216] true {r_ok:.3e}  bf16 weights {r_bf16:.3e} ({r_bf16 / BARS["gemm"]:.0f}x the bar)')
    assert r_ok <= BARS['gemm']
    assert r_bf16 >= 10 * BARS['gemm'], r_bf16


@pytest.mark.parametrize('arch', ARCHS)
def test_end_to_end_matches_reference(models, gold, arch):
    m = model_of(models, arch)
    u8 = synthetic.make_structured_crops_u8(GOLD_FACES, seed=GOLD_SEED).to(DEV)
    x = synthetic.normalize_crops(u8)
    eng = m._engine(DEV)
    out, pool = eng.forward_resnet(x)
    lmk = m.forward_landmarks(x)
    e_out = rp.max_rel_err(out.cpu().numpy(), gold[f'{arch}_out102'])
    e_lmk = rp.max_rel_err(lmk.cpu().numpy(), gold[f'{arch}_lmk'])
    print(f'\n[{arch}] out102 err {e_out:.3e}  landmarks err {e_lmk:.3e}')
    assert e_out < E2E_TOL and e_lmk < E2E_TOL
    assert pool.shape == (GOLD_FACES, m.I2P.backbone.feature_dim)
    out_u8, pool_u8 = eng.forward_resnet(u8)                           # (v - 127.5) / 128 in the stem: the same bits
    assert same_bits(out_u8, out) and same_bits(pool_u8, pool)
    again, _ = eng.forward_resnet(x)
    assert same_bits(again, out)
    params, feat = m.I2P.forward_test(x)
    assert same_bits(params, out[:, :62]) and same_bits(feat, pool)
    with pytest.raises(Exception, match='use syn_resnet_forward'):
        eng.forward_resnet50(x)
    assert eng.poll_error() == 0


@pytest.mark.parametrize('arch', ('resnet18', 'resnet101'))
def test_ragged_batches_are_bit_identical_per_face(models, arch):
    eng = model_of(models, arch)._engine(DEV)
    big = 1100
    u8 = torch.cat([synthetic.make_structured_crops_u8(16, seed=8), synthetic.make_crops_u8(big - 16, seed=8)]).to(DEV)
    x = synthetic.normalize_crops(u8)
    full, pool = eng.forward_resnet(x)
    for b in (1, 2, 7, 129):
        for f0 in (0, big - b):
            o, p = eng.forward_resnet(x[f0:f0 + b])
            assert same_bits(o, full[f0:f0 + b]) and same_bits(p, pool[f0:f0 + b]), (b, f0)
    assert eng.poll_error() == 0


def test_resnet50_generic_entry_point_is_bit_identical(synth_pack):
    """syn_resnet_forward and syn_resnet50_forward run the same launches on a resnet50 handle: the same bits, and the
    uint8 crops give the bits of their normalised copy."""
    m = make_model(synth_resnet.build_resnet_state_dict(0, 'resnet50'), 'resnet50', strict=False)
    eng = m._engine(DEV)
    u8 = synthetic.make_structured_crops_u8(19, seed=12).to(DEV)
    x = synthetic.normalize_crops(u8)
    a, pa = eng.forward_resnet50(x)
    b, pb = eng.forward_resnet(x)
    c, pc = eng.forward_resnet(u8)
    assert same_bits(a, b) and same_bits(pa, pb) and same_bits(a, c) and same_bits(pa, pc)
    assert eng.poll_error() == 0


def test_reference_caller_sequences(synth_pack, gold):
    """SynergyNet(args) with args.arch='resnet101' driven the way the reference's scripts drive it."""
    from synergynet_b200 import model_building
    arch = 'resnet101'
    sd0 = checkpoint(arch)
    model = model_building.SynergyNet(types.SimpleNamespace(arch=arch, img_size=120, devices_id=[0]))
    dp = nn.DataParallel(model, device_ids=[0])
    res = dp.load_state_dict({'module.I2P.backbone.' + k: v for k, v in sd0.items()}, strict=False)
    assert not [k for k in res.missing_keys if k.startswith('module.I2P.')] and not res.unexpected_keys
    dp.eval()
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(GOLD_FACES, seed=GOLD_SEED))
    params = dp.module.forward_test(x.to(DEV))
    assert rp.max_rel_err(params.cpu().numpy(), gold[f'{arch}_out102'][:, :62]) < E2E_TOL
    p_cpu = model.forward_test(x)                                          # CPU tensor in, CPU tensor out
    assert not p_cpu.is_cuda and same_bits(p_cpu, params.cpu())
    lmk = model.reconstruct_vertex_62(params)
    assert rp.max_rel_err(lmk.cpu().numpy(), gold[f'{arch}_lmk']) < E2E_TOL
    # a new checkpoint in the same model rebuilds the engine; the old one back gives the old bits
    sd1 = checkpoint(arch, 1)
    model.load_state_dict({'I2P.backbone.' + k: v for k, v in sd1.items()}, strict=False)
    p1 = model.forward_test(x.to(DEV))
    want1, _ = resnets64.resnet_forward({'I2P.backbone.' + k: v for k, v in sd1.items()}, x, arch)
    assert rp.max_rel_err(p1.cpu().numpy(), want1[:, :62].numpy()) < E2E_TOL and not same_bits(p1, params)
    model.load_state_dict({'I2P.backbone.' + k: v for k, v in sd0.items()}, strict=False)
    assert same_bits(model.forward_test(x.to(DEV)), params)
    with pytest.raises(RuntimeError, match='1280-d image feature'):
        model(x.to(DEV), params)
    assert model._engine(DEV).poll_error() == 0


@pytest.mark.parametrize('arch', ('resnet18', 'resnet50'))
def test_get_all_outputs_runs_the_resnet(synth_pack, arch):
    """get_all_outputs on a 3-face scene equals forward_test on the host-made crops (crop_img + cv2.resize) followed by
    reconstruct_image / pose_decode: the ResNet runs on the device-made uint8 crops."""
    from golden import make_golden_resize as gr
    import cv2
    from synergynet_b200.inference import INTER_LANCZOS4, roi_affine, square_roi
    model = make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
    scene = synthetic.make_scene_u8(360, 480, 4)
    rects = [[60.3, 80.1, 200.9, 250.4, 0.98], [250.2, -20.0, 372.6, 140.7, 0.91], [300.0, 150.0, 470.0, 350.0, 0.9]]
    lmk_a, mesh_a, pose_a = model.get_all_outputs(scene.copy(), rects=rects)
    boxes = [square_roi(list(r)) for r in rects]
    crops = np.stack([cv2.resize(gr.host_crop(scene, b), dsize=(120, 120), interpolation=INTER_LANCZOS4) for b in boxes])
    xc = synthetic.normalize_crops(torch.from_numpy(crops).permute(0, 3, 1, 2).contiguous())
    p = model.forward_test(xc.to(DEV))
    eng = model._engine(DEV)
    roi5 = torch.from_numpy(roi_affine(boxes)).to(DEV)
    want_lmk = eng.reconstruct_image(p, roi5, dense=False).cpu().numpy()
    want_mesh = eng.reconstruct_image(p, roi5, dense=True).cpu().numpy()
    ang, t3d = eng.pose_decode(p, roi5)
    assert np.array_equal(np.stack(lmk_a), want_lmk) and np.array_equal(np.stack(mesh_a), want_mesh)
    assert np.array_equal(np.array([q[0] for q in pose_a]), ang.cpu().numpy())
    assert np.array_equal(np.array([q[1] for q in pose_a]), t3d.cpu().numpy())
    assert eng.poll_error() == 0


def test_mobilenet_v2_unchanged_by_a_resnet_model(synth_pack):
    """A mobilenet_v2 model's landmarks on the same device are bit-identical before and after a wide_resnet101_2 model
    is created and run in the same process."""
    from oracle import synth_model
    m2 = make_model(synth_model.build_state_dict(0))
    x = seeded_crops(9, 3)
    before = m2.forward_landmarks(x).clone()
    m1 = make_model(checkpoint('wide_resnet101_2'), 'wide_resnet101_2', strict=False)
    m1.forward_landmarks(seeded_crops(130, 4))
    torch.cuda.synchronize()
    assert same_bits(m2.forward_landmarks(x), before)


@pytest.mark.parametrize('arch', ('resnet18', 'resnet152', 'wide_resnet50_2'))
def test_launches_and_timing_names(models, arch):
    """One timing entry per launch, in plan order: stem, max-pool, each block's inner convs, its downsample, the conv that
    adds the shortcut, then the pool and the heads."""
    eng = model_of(models, arch)._engine(DEV)
    n = len(resnets64.conv_keys(arch))
    basic = backbone.RESNET_ARCHS[arch][0] < 50
    want = ['resnet_stem_kernel', 'maxpool3x3s2_kernel']
    for inner, last, ds in resnets64.blocks(arch):
        want += ['resnet_conv3x3'] if basic else ['resnet_conv1x1_a', 'resnet_conv3x3']
        want += ['resnet_downsample'] if ds is not None else []
        want += ['resnet_conv3x3_res' if basic else 'resnet_conv1x1_b']
    want += ['avgpool_kernel', 'resnet_heads']
    assert len(want) == n + 3
    eng.set_timing(True)
    n0 = eng.launch_count
    eng.forward_resnet(seeded_crops(3, 2))
    torch.cuda.synchronize()
    launches = eng.launch_count - n0
    names = [nm for nm, _ in eng.timings(max_entries=256)]
    eng.set_timing(False)
    assert launches == n + 3 and names == want
    assert eng.poll_error() == 0


def test_backbone_entry_points_reject_65536_faces(synth_pack):
    """All five forward and debug entry points of the conv+BN backbones refuse 65536 faces with SYN_ERR_INVALID before
    they launch anything (the bound dw3x3_kernel's grid.y sets, shared by every entry point)."""
    from oracle import synth_mbv1
    rn = make_model(synth_resnet.build_resnet_state_dict(0, 'resnet50'), 'resnet50', strict=False)._engine(DEV)
    v1 = make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, 'mobilenet_025'), 'mobilenet_025', strict=False)._engine(DEV)
    x = torch.zeros((1, 3, 120, 120), device=DEV)
    out = torch.empty((1, 2048), device=DEV)
    rm = torch.zeros((1,), device=DEV, dtype=torch.int32)
    b = 65536
    calls = [(rn, lambda L, h: L.syn_resnet50_forward(h, x.data_ptr(), b, out.data_ptr(), out.data_ptr(), None)),
             (rn, lambda L, h: L.syn_resnet_forward(h, x.data_ptr(), 0, b, out.data_ptr(), out.data_ptr(), None)),
             (rn, lambda L, h: L.syn_debug_resnet_until(h, x.data_ptr(), b, 2, out.data_ptr(), rm.data_ptr(), None)),
             (v1, lambda L, h: L.syn_mbv1_forward(h, x.data_ptr(), 0, b, out.data_ptr(), out.data_ptr(), None)),
             (v1, lambda L, h: L.syn_debug_mbv1_until(h, x.data_ptr(), b, 1, out.data_ptr(), rm.data_ptr(), None))]
    for i, (eng, call) in enumerate(calls):
        n0 = eng.launch_count
        assert call(eng._lib, eng._h) == 1, i                                     # SYN_ERR_INVALID
        assert b'65535' in eng._lib.syn_last_error(), i
        assert eng.launch_count == n0, i
    rn.forward_resnet50(x)                                          # both handles still run
    v1.forward_mobilenet_v1(x)
    torch.cuda.synchronize()
    assert rn.poll_error() == 0 and v1.poll_error() == 0
