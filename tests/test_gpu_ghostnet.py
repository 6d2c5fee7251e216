"""The GhostNet backbone on the H100: every stage against the float64 oracle (oracle/ghost64.py), element by element, then
end to end against the reference module's golden output, and through the module's forward, CUDA graphs, poisoned
workspaces and two threads.

Each stage is fed the GPU's own outputs of the stages it reads and held to |got - want| <= TAU * S; every row maximum a
stage records is compared bit for bit.  The batches put the last 128-row tile of every map size, and of the per-face
SE and head GEMMs, in each of its shapes (ghost64.check_ghost_batches); the faces checked include the last face and the
faces around the last tile's edge.
"""
import os

import numpy as np
import pytest
import torch

from oracle import gemm64, ghost64, synth_ghost
from oracle import reference_port as rp
from oracle.stage_check import TOL, Ratios, check_rowmax, face_picker, report, same_bits, seeded_crops
from synergynet_b200 import backbone, synthetic

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
BARS = ghost64.TAU
GOLD_FACES, GOLD_SEED = 4, 31             # tests/golden/make_golden_ghostnet.py


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ref_vectors_ghostnet.npz'), allow_pickle=False))


def _module(sd):
    m = backbone.ghostnet()
    m.load_state_dict(sd, strict=True)
    return m.eval()


@pytest.fixture(scope='module')
def model(synth_pack):
    return _module(synth_ghost.build_ghostnet_state_dict(0))


def ghost_ratios(eng, sd, x, faces, ratios):
    """Run every stage on batch ``x`` and hold the given faces to the oracle; row maxima bit for bit."""
    nf = len(faces)
    pick, where = face_picker(x.shape[0], faces, x.device)
    outs = {-1: x[faces].cpu()}
    for s, st in enumerate(ghost64.stage_table()):
        out, rm = eng.debug_ghostnet_until(x, s)
        assert out.shape == (x.shape[0] * st['rows'], st['cols']), s
        if st['rowmax']:
            check_rowmax(out, rm, f'stage {s} {st["op"]}')
        else:
            assert rm is None
        got = pick(out)
        kind = ghost64.kind(st['op'])
        ratios.add(kind, f'{st["op"]}{s}', got, ghost64.stage(sd, s, outs, nf), where(st['rows']))
        outs[s] = got
    assert eng.poll_error() == 0
    assert eng.poll_saturation(warn=False) == 0


def test_stage_plan_matches_the_oracle(model):
    eng = model._engine(DEV)
    assert eng._lib.syn_ghost_num_stages() == ghost64.NUM_STAGES
    for s, st in enumerate(ghost64.stage_table()):
        assert eng.ghostnet_stage_desc(s) == (st['rows'], st['cols'], st['rowmax']), s


@pytest.mark.parametrize('batch', ghost64.BATCHES)
def test_every_stage_matches_float64_oracle(model, batch):
    ghost64.check_ghost_batches()
    sd = synth_ghost.build_ghostnet_state_dict(0)
    ratios = Ratios()
    ghost_ratios(model._engine(DEV), sd, seeded_crops(batch, 700 + batch), ghost64.faces(batch), ratios)
    report(f'ghostnet B={batch}', ratios)
    bad = ghost64.over(ratios)
    assert not bad, bad


def test_rescaled_checkpoint(synth_pack, gold):
    """Hidden channels spread over 2^10: the same function (out102 of the reference within TOL) and every stage under the
    same bar, with the GEMMs' row scales spread as widely."""
    sd = synth_ghost.reparametrize_ghostnet(synth_ghost.build_ghostnet_state_dict(0), **ghost64.WIDE)
    eng = _module(sd)._engine(DEV)
    out, _ = eng.forward_ghostnet(seeded_crops(GOLD_FACES, GOLD_SEED))
    err = rp.max_rel_err(out.cpu().numpy(), gold['ghostnet_out102'])
    print(f'\n[ghostnet rescaled] out102 err {err:.3e}')
    assert err < TOL
    batch = 33
    ratios = Ratios()
    ghost_ratios(eng, sd, seeded_crops(batch, 700 + batch), ghost64.faces(batch), ratios)
    report(f'ghostnet rescaled B={batch}', ratios)
    bad = ghost64.over(ratios)
    assert not bad, bad


def _stage_of(op, block):
    return next(s for s, st in enumerate(ghost64.stage_table()) if st['op'] == op and st['block'] == block)


def test_negative_controls_fail_the_bar(model):
    """ghost2's primary GEMM of block 9 and the SE conv_reduce of block 10, on the GPU's own inputs through the same
    GEMM: with the true row maxima they pass; with their weights rounded to bf16, or with rowmax_in / 8 (the scaled row
    leaves the fp16 range and is clamped), they must fail by a wide margin."""
    sd = synth_ghost.build_ghostnet_state_dict(0)
    eng = model._engine(DEV)
    x = seeded_crops(2, 5)
    b9, b10 = ghost64.blocks()[9], ghost64.blocks()[10]
    w, bias = ghost64._bn(sd, b9['p'] + 'ghost2.primary_conv.0', b9['p'] + 'ghost2.primary_conv.1')
    wr, br, _, _ = ghost64.se_weights(sd, b10)
    cases = [('ghost primary', _stage_of('primary2', 9) - 1, w.reshape(w.shape[0], -1), bias, 0),
             ('SE reduce', _stage_of('se_reduce', 10) - 1, wr, br, 2)]
    for tag, src, wt, bt, act in cases:
        a, rm = eng.debug_ghostnet_until(x, src)
        assert rm is not None
        want = gemm64.gemm(a.cpu(), wt, bt, act == 2)
        ratio = lambda weights, rmax: gemm64.worst(eng.debug_gemm(weights, bt.float(), a, rmax, act=act)[0].cpu(), *want)[0]
        wf = wt.float()
        r_ok = ratio(wf, rm)
        r_bf16 = ratio(wf.bfloat16().float(), rm)
        r_div8 = ratio(wf, (rm.view(torch.float32) / 8).view(torch.int32))
        print(f'\n[negative controls, {tag}] true {r_ok:.3e}  bf16 weights {r_bf16:.3e} ({r_bf16 / BARS["gemm"]:.0f}x the bar)'
              f'  rowmax/8 {r_div8:.3e} ({r_div8 / BARS["gemm"]:.0f}x the bar)')
        assert r_ok <= BARS['gemm']
        assert r_bf16 >= 10 * BARS['gemm'] and r_div8 >= 10 * BARS['gemm'], (tag, r_bf16, r_div8)
        assert eng.poll_saturation(warn=False) == 1          # the clamps of the rowmax / 8 run are flagged, and cleared


def test_end_to_end_matches_reference(model, gold):
    u8 = synthetic.make_structured_crops_u8(GOLD_FACES, seed=GOLD_SEED).to(DEV)
    x = synthetic.normalize_crops(u8)
    eng = model._engine(DEV)
    out, feat = eng.forward_ghostnet(x)
    err = rp.max_rel_err(out.cpu().numpy(), gold['ghostnet_out102'])
    print(f'\n[ghostnet] out102 err {err:.3e}')
    assert err < TOL
    assert feat.shape == (GOLD_FACES, 1280) and float(feat.min()) >= 0.0
    out_u8, feat_u8 = eng.forward_ghostnet(u8)                       # (v - 127.5) / 128 in the stem: the same bits
    assert same_bits(out_u8, out) and same_bits(feat_u8, feat)
    again, _ = eng.forward_ghostnet(x)
    assert same_bits(again, out)
    assert same_bits(model(x), out)                                   # the module's forward is the engine's
    cpu = model(x.cpu())                                              # CPU in, CPU out
    assert not cpu.is_cuda and same_bits(cpu, out.cpu())
    assert eng.poll_error() == 0


def test_module_refusals(model):
    with pytest.raises(RuntimeError, match='eval'):
        backbone.ghostnet().train()(torch.zeros(1, 3, 120, 120, device=DEV))
    with pytest.raises(RuntimeError, match='120'):
        model(torch.zeros(1, 3, 112, 112, device=DEV))


def test_ragged_batches_are_bit_identical_per_face(model):
    eng = model._engine(DEV)
    big = 1100
    u8 = torch.cat([synthetic.make_structured_crops_u8(16, seed=8), synthetic.make_crops_u8(big - 16, seed=8)]).to(DEV)
    x = synthetic.normalize_crops(u8)
    full, feat = eng.forward_ghostnet(x)
    for b in (1, 2, 7, 129):
        for f0 in (0, big - b):
            o, f = eng.forward_ghostnet(x[f0:f0 + b])
            assert same_bits(o, full[f0:f0 + b]) and same_bits(f, feat[f0:f0 + b]), (b, f0)
    assert eng.poll_error() == 0


def test_graph_replay_and_capture_refusal(synth_pack):
    from test_gpu_graph_replay import K, _flags_clear, refused, replay_case
    eng = _module(synth_ghost.build_ghostnet_state_dict(0))._engine(DEV)      # a handle whose workspace holds 128 faces
    for b in (128, 13):
        for dtype in ('fp32', 'uint8'):
            u8 = [synthetic.make_structured_crops_u8(b, seed=300 + 7 * r + b).to(DEV) for r in range(K + 1)]
            ins = [(u if dtype == 'uint8' else synthetic.normalize_crops(u),) for u in u8]
            replay_case(f'ghostnet B={b} {dtype}', eng, eng.forward_ghostnet, ins)
    big = synthetic.normalize_crops(synthetic.make_structured_crops_u8(300, seed=4)).to(DEV)
    refused('ghostnet growth', lambda: eng.forward_ghostnet(big), 'syn_ghost_forward', 'workspace')
    _flags_clear(eng)


def test_poisoned_workspaces_and_outputs(model):
    from test_gpu_poison import _crops, _snap, check_cases
    eng = model._engine(DEV)
    cases = {}
    for b in (13, 19, 128):
        u8 = _crops(b, 300 + b).to(DEV)
        for dt, x in (('uint8', u8), ('fp32', synthetic.normalize_crops(u8))):
            cases[f'ghostnet B={b} {dt}'] = lambda x=x: eng.forward_ghostnet(x)
    r0 = {n: _snap(fn()) for n, fn in cases.items()}
    eng.forward_ghostnet(synthetic.normalize_crops(_crops(160, 11)).to(DEV))
    check_cases(cases, r0, [eng], [eng])


def test_two_threads_on_two_streams(model):
    from test_gpu_concurrency import ITERS, run_threads
    eng = model._engine(DEV)
    xs = [synthetic.normalize_crops(synthetic.make_structured_crops_u8(b, seed=90 + b)).to(DEV) for b in (16, 96)]
    want = [[o.clone() for o in eng.forward_ghostnet(x)] for x in xs]
    m2 = _module(synth_ghost.build_ghostnet_state_dict(0))
    run2 = m2._engine(DEV).forward_ghostnet
    got = run_threads(lambda t, i: [o.clone() for o in run2(xs[t])])
    for t in range(2):
        for i in range(ITERS):
            assert all(same_bits(g, w) for g, w in zip(got[t][i], want[t])), f'thread {t} iteration {i}'
    assert m2._engine(DEV).poll_error() == 0


def test_mobilenet_v2_unchanged_by_a_ghostnet_model(synth_pack):
    """A mobilenet_v2 model's landmarks on the same device are bit-identical before and after a GhostNet model is created
    and run in the same process."""
    from oracle import synth_model
    from oracle.stage_check import make_model
    m2 = make_model(synth_model.build_state_dict(0))
    x = seeded_crops(9, 3)
    before = m2.forward_landmarks(x).clone()
    g = _module(synth_ghost.build_ghostnet_state_dict(1))
    g(seeded_crops(130, 4))
    torch.cuda.synchronize()
    assert same_bits(m2.forward_landmarks(x), before)


def test_timing_names(model):
    eng = model._engine(DEV)
    eng.set_timing(True)
    eng.forward_ghostnet(seeded_crops(3, 2))
    names = [n for n, _ in eng.timings(256)]
    eng.set_timing(False)
    label = {'stem': 'ghost_stem_kernel', 'primary1': 'ghost_primary', 'primary2': 'ghost_primary', 'ghost1': 'ghost_cheap',
             'ghost2': 'ghost_cheap_add', 'dw': 'ghost_dw', 'se_pool': 'ghost_se_pool', 'se_reduce': 'ghost_se_reduce',
             'se_expand': 'ghost_se_expand', 'se_apply': 'ghost_se_apply', 'sc_dw': 'ghost_shortcut_dw',
             'sc_pw': 'ghost_shortcut_pw', 'conv_bn_act': 'ghost_conv_bn_act', 'pool': 'ghost_avgpool',
             'conv_head': 'ghost_conv_head', 'heads': 'ghost_heads'}
    assert names == [label[st['op']] for st in ghost64.stage_table()]


def test_65536_faces_are_refused_before_any_launch(model):
    eng = model._engine(DEV)
    x = torch.zeros((1, 3, 120, 120), device=DEV)
    out = torch.empty((1, 1280), device=DEV)
    rm = torch.zeros((1,), device=DEV, dtype=torch.int32)
    b = 65536
    for i, call in enumerate((lambda L, h: L.syn_ghost_forward(h, x.data_ptr(), 0, b, out.data_ptr(), out.data_ptr(), None),
                              lambda L, h: L.syn_debug_ghost_until(h, x.data_ptr(), b, 1, out.data_ptr(), rm.data_ptr(), None))):
        n0 = eng.launch_count
        assert call(eng._lib, eng._h) == 1, i                                     # SYN_ERR_INVALID
        assert b'65535' in eng._lib.syn_last_error(), i
        assert eng.launch_count == n0, i
    eng.forward_ghostnet(x)
    torch.cuda.synchronize()
    assert eng.poll_error() == 0
