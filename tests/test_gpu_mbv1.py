"""The MobileNetV1 backbones on the H100: every stage of every width against the float64 oracle (oracle/mbv1_64.py),
element by element, then end to end against the reference module's golden outputs and through the reference's caller
sequences.

Each stage is fed the GPU's own output of the previous stage and held to |got - want| <= TAU * S; every row maximum a
stage records is compared bit for bit.  The batches put the last 128-row tile of every map size in each of its shapes
(mbv1_64.check_mbv1_batches); the faces checked include the last face and the faces around the last tile's edge.
"""
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import gemm64, mbv1_64, synth_mbv1
from oracle import reference_port as rp
from oracle.stage_check import (TAU, TOL, WIDE, Ratios, check_rowmax, face_picker, make_model, over, report, same_bits,
                                seeded_crops)
from synergynet_b200 import backbone, synthetic

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
ARCHS = tuple(backbone.MBV1_WIDTHS)
BARS = TAU['mbv1_64']
GOLD_FACES, GOLD_SEED = 4, 31             # tests/golden/make_golden_mbv1.py


@pytest.fixture(scope='module')
def gold():
    import os
    return dict(np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_vectors_mbv1.npz'), allow_pickle=False))


@pytest.fixture(scope='module')
def models(synth_pack):
    return {a: make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, a), a, strict=False) for a in ARCHS}


def mbv1_ratios(eng, sd, x, faces, ratios):
    """Run every stage on batch ``x`` and hold the given faces to the oracle; row maxima bit for bit."""
    nf = len(faces)
    pick, where = face_picker(x.shape[0], faces, x.device)
    inp = x[faces].cpu()
    for s in range(mbv1_64.NUM_STAGES):
        out, rm = eng.debug_mobilenet_v1_until(x, s)
        if s in (0, 26, 27) or (s <= 26 and s % 2 == 1):
            check_rowmax(out, rm, f'stage {s}')
        else:
            assert rm is None
        got = pick(out)
        kind = 'dw' if s == 0 or (s <= 26 and s % 2 == 1) else 'pool' if s == 27 else 'gemm'
        ratios.add(kind, s, got, mbv1_64.stage(sd, s, inp, nf), where(got.shape[0] // nf))
        inp = got
    assert eng.poll_error() == 0


@pytest.mark.parametrize('batch', mbv1_64.BATCHES)
@pytest.mark.parametrize('arch', ARCHS)
def test_every_stage_matches_float64_oracle(models, arch, batch):
    mbv1_64.check_mbv1_batches()
    sd = synth_mbv1.build_mobilenet_v1_state_dict(0, arch)
    eng = models[arch]._engine(DEV)
    ratios = Ratios()
    mbv1_ratios(eng, sd, seeded_crops(batch, 700 + batch), mbv1_64.faces(batch), ratios)
    report(f'{arch} B={batch}', ratios)
    bad = over('mbv1_64', ratios)
    assert not bad, bad


@pytest.mark.parametrize('arch', ARCHS)
def test_rescaled_checkpoint(synth_pack, gold, arch):
    """Hidden channels spread over 2^10: the same function (out102 of the reference within TOL) and every stage under the
    same bar, with the GEMMs' row scales spread as widely."""
    sd = synth_mbv1.reparametrize_mobilenet_v1(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), **WIDE['mbv1_64'])
    m = make_model(sd, arch, strict=False)
    eng = m._engine(DEV)
    out, _ = eng.forward_mobilenet_v1(seeded_crops(GOLD_FACES, GOLD_SEED))
    err = rp.max_rel_err(out.cpu().numpy(), gold[f'{arch}_out102'])
    print(f'\n[{arch} rescaled] out102 err {err:.3e}')
    assert err < TOL
    batch = 33
    ratios = Ratios()
    mbv1_ratios(eng, sd, seeded_crops(batch, 700 + batch), mbv1_64.faces(batch), ratios)
    report(f'{arch} rescaled B={batch}', ratios)
    bad = over('mbv1_64', ratios)
    assert not bad, bad


def test_negative_controls_fail_the_bar(models):
    """conv_sep of dw5_1 on the GPU's own depthwise output through the same GEMM: with the true row maxima it passes;
    with its weights rounded to bf16, or with rowmax_in / 8 (the scaled row leaves the fp16 range and is clamped), it
    must fail by a wide margin."""
    arch, batch, idx = 'mobilenet_1', 2, 14
    sd = synth_mbv1.build_mobilenet_v1_state_dict(0, arch)
    eng = models[arch]._engine(DEV)
    x = seeded_crops(batch, 5)
    a, rm = eng.debug_mobilenet_v1_until(x, idx - 1)
    w4, b = mbv1_64.fold(sd, idx)
    w = w4.reshape(w4.shape[0], -1).float()
    want = mbv1_64.pointwise(sd, idx, a.cpu())
    ratio = lambda weights, rmax: gemm64.worst(eng.debug_gemm(weights, b.float(), a, rmax, act=2)[0].cpu(), *want)[0]
    r_ok = ratio(w, rm)
    r_bf16 = ratio(w.bfloat16().float(), rm)
    r_div8 = ratio(w, (rm.view(torch.float32) / 8).view(torch.int32))
    print(f'\n[negative controls] true {r_ok:.3e}  bf16 weights {r_bf16:.3e} ({r_bf16 / BARS["gemm"]:.0f}x the bar)  '
          f'rowmax/8 {r_div8:.3e} ({r_div8 / BARS["gemm"]:.0f}x the bar)')
    assert r_ok <= BARS['gemm']
    assert r_bf16 >= 10 * BARS['gemm'] and r_div8 >= 10 * BARS['gemm'], (r_bf16, r_div8)


@pytest.mark.parametrize('arch', ARCHS)
def test_end_to_end_matches_reference(models, gold, arch):
    m = models[arch]
    u8 = synthetic.make_structured_crops_u8(GOLD_FACES, seed=GOLD_SEED).to(DEV)
    x = synthetic.normalize_crops(u8)
    eng = m._engine(DEV)
    out, pool = eng.forward_mobilenet_v1(x)
    lmk = m.forward_landmarks(x)
    e_out = rp.max_rel_err(out.cpu().numpy(), gold[f'{arch}_out102'])
    e_lmk = rp.max_rel_err(lmk.cpu().numpy(), gold[f'{arch}_lmk'])
    print(f'\n[{arch}] out102 err {e_out:.3e}  landmarks err {e_lmk:.3e}')
    assert e_out < TOL and e_lmk < TOL
    assert pool.shape == (GOLD_FACES, int(1024 * backbone.MBV1_WIDTHS[arch]))
    out_u8, pool_u8 = eng.forward_mobilenet_v1(u8)                     # (v - 127.5) / 128 in the stem: the same bits
    assert same_bits(out_u8, out) and same_bits(pool_u8, pool)
    again, _ = eng.forward_mobilenet_v1(x)
    assert same_bits(again, out)
    params = m.forward_test(x)
    assert same_bits(params, out[:, :62])
    assert eng.poll_error() == 0


@pytest.mark.parametrize('arch', ('mobilenet_1', 'mobilenet_025'))
def test_ragged_batches_are_bit_identical_per_face(models, arch):
    eng = models[arch]._engine(DEV)
    big = 1100
    u8 = torch.cat([synthetic.make_structured_crops_u8(16, seed=8), synthetic.make_crops_u8(big - 16, seed=8)]).to(DEV)
    x = synthetic.normalize_crops(u8)
    full, pool = eng.forward_mobilenet_v1(x)
    for b in (1, 2, 7, 129):
        for f0 in (0, big - b):
            o, p = eng.forward_mobilenet_v1(x[f0:f0 + b])
            assert same_bits(o, full[f0:f0 + b]) and same_bits(p, pool[f0:f0 + b]), (b, f0)
    assert eng.poll_error() == 0


def test_reference_caller_sequences(synth_pack, gold):
    """SynergyNet(args) with args.arch='mobilenet_1' driven the way the reference's scripts drive it."""
    from golden import make_golden_resize as gr
    import cv2
    from synergynet_b200 import model_building
    from synergynet_b200.inference import INTER_LANCZOS4, roi_affine, square_roi
    arch = 'mobilenet_1'
    sd0 = synth_mbv1.build_mobilenet_v1_state_dict(0, arch)
    model = model_building.SynergyNet(types.SimpleNamespace(arch=arch, img_size=120, devices_id=[0]))
    dp = nn.DataParallel(model, device_ids=[0])
    res = dp.load_state_dict({'module.I2P.backbone.' + k: v for k, v in sd0.items()}, strict=False)
    assert not [k for k in res.missing_keys if k.startswith('module.I2P.')] and not res.unexpected_keys
    dp.eval()
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(GOLD_FACES, seed=GOLD_SEED))
    params = dp.module.forward_test(x.to(DEV))
    assert rp.max_rel_err(params.cpu().numpy(), gold[f'{arch}_out102'][:, :62]) < TOL
    p_cpu = model.forward_test(x)                                          # CPU tensor in, CPU tensor out
    assert not p_cpu.is_cuda and same_bits(p_cpu, params.cpu())
    lmk = model.reconstruct_vertex_62(params)
    assert rp.max_rel_err(lmk.cpu().numpy(), gold[f'{arch}_lmk']) < TOL
    # a new checkpoint in the same model rebuilds the engine; the old one back gives the old bits
    sd1 = synth_mbv1.build_mobilenet_v1_state_dict(1, arch)
    model.load_state_dict({'I2P.backbone.' + k: v for k, v in sd1.items()}, strict=False)
    p1 = model.forward_test(x.to(DEV))
    want1, _ = mbv1_64.forward64(sd1, x)
    assert rp.max_rel_err(p1.cpu().numpy(), want1[:, :62].numpy()) < TOL and not same_bits(p1, params)
    model.load_state_dict({'I2P.backbone.' + k: v for k, v in sd0.items()}, strict=False)
    assert same_bits(model.forward_test(x.to(DEV)), params)
    with pytest.raises(RuntimeError, match='1280-d image feature'):
        model(x.to(DEV), params)
    # get_all_outputs: this backbone on the device-made uint8 crops, then the image-space stages
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


def test_mobilenet_v2_unchanged_by_a_mobilenet_v1_model(synth_pack):
    """A mobilenet_v2 model's landmarks on the same device are bit-identical before and after a MobileNetV1 model is
    created and run in the same process."""
    from oracle import synth_model
    m2 = make_model(synth_model.build_state_dict(0))
    x = seeded_crops(9, 3)
    before = m2.forward_landmarks(x).clone()
    m1 = make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, 'mobilenet_2'), 'mobilenet_2', strict=False)
    m1.forward_landmarks(seeded_crops(130, 4))
    torch.cuda.synchronize()
    assert same_bits(m2.forward_landmarks(x), before)


def test_timing_names(models):
    eng = models['mobilenet_05']._engine(DEV)
    eng.set_timing(True)
    eng.forward_mobilenet_v1(seeded_crops(3, 2))
    names = [n for n, _ in eng.timings()]
    eng.set_timing(False)
    assert names == (['mbv1_stem_kernel'] + ['mbv1_dw3x3', 'mbv1_conv_sep'] * 12 + ['mbv1_dw3x3', 'mbv1_conv_sep_last',
                                                                                     'mbv1_avgpool', 'mbv1_heads'])
