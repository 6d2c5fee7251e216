"""Every face of production-size MobileNetV2 batches, bit for bit, against a pool of faces held to the float64 oracle.

A pool of P = 64 distinct crops is run at B = P and every pool face is held to ``block64`` stage by stage
(``stage_check.stage_ratios``).  Larger batches are then made of pool faces only -- face b is pool face
(b + b // P) % P (``tile_cover.placement``), so each repetition shifts the pool by one face -- and every face of every
output must carry the bits of its pool face: params, pooled feature and landmarks of every device entry point, every
block output of the fused engine, every conv of the unfused engines, and the host pipelines (submitted and blocking,
multi-chunk).  Every kernel of the backbone computes a face from that face's rows alone in a fixed per-element order
(its only atomics are maxima), so a face's bits must not depend on the tile, slot or chunk it lands in; a race or a
tile-plan slip anywhere in the batch shows up as a face that differs.

The same file checks the centre-crop frame of every uint8 stem against crops framed on the host, and the frame batch of
the detector at its 64-frame limit.  H100 only.
"""
import numpy as np
import pytest
import torch

from oracle import synth_mbv1, synth_model, synth_resnet, tile_cover
from oracle.stage_check import ENGINES, Ratios, make_model, over, report, stage_ratios
from synergynet_b200 import _lib, faceboxes, synthetic
from synergynet_b200.backbone import conv_plan

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
P = 64                       # pool faces
POOL_SEED = 4242
BENCH_BATCH = 1024           # bench.py's batch
ORACLE_CHUNK = 32            # pool faces per float64 pass (bounds the host memory of the 52 conv outputs)


# ---- helpers ---------------------------------------------------------------------------------------------------------
def _i32(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(t.shape[0], -1).view(torch.int32)


def differing_faces(got: torch.Tensor, pool_out: torch.Tensor, place: torch.Tensor):
    """The faces b of a batch output (first axis = face) whose bits differ from those of pool face ``place[b]`` in the
    pool's output of the same stage."""
    want = _i32(pool_out.to(got.device)).index_select(0, place.to(got.device))
    return (_i32(got) != want).any(1).nonzero().flatten().tolist()


def _assert_same(name, got, pool_out, place):
    bad = differing_faces(got, pool_out, place)
    assert not bad, f'{name}: {len(bad)} of {got.shape[0]} faces differ from their pool face, first {bad[:8]}'


def _engine(model, kind):
    model.set_engine(kind)
    return model._engine(DEV)


def framed(u8: torch.Tensor, m: int) -> torch.Tensor:
    """CenterCrop(m, mode='test') of the reference loader on the raw pixels: ``img[:, m:h-m, m:w-m]`` into zeros
    (utils/ddfa.py:231,239)."""
    out = torch.zeros_like(u8)
    out[:, :, m:120 - m, m:120 - m] = u8[:, :, m:120 - m, m:120 - m]
    return out


@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def model(synth_pack, sd):
    return make_model(sd)


@pytest.fixture(scope='module')
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope='module')
def pool_u8():
    return synthetic.make_structured_crops_u8(P, seed=POOL_SEED)


@pytest.fixture(scope='module')
def batches(sms):
    """B = 1024 and the three tile-cover batches; together they meet every placement claim on this device."""
    out = {'bench': BENCH_BATCH, **tile_cover.choose_batches(sms)}
    met_any, claims = set(), set()
    for kind, b in out.items():
        if kind != 'bench':
            tile_cover.check_plan(kind, b, sms)
        met, dropped = tile_cover.check_placement(b, sms, P)
        met_any |= set(met)
        claims |= set(met) | set(dropped)
        print(f'\n[placement {kind} B={b}] dropped: {dropped}')
    assert met_any == claims, claims - met_any
    return out


def pool_outputs(eng, u8: torch.Tensor):
    """(params, pooled feature, landmarks) of the pool at B = P through every device entry point, which must agree."""
    x = synthetic.normalize_crops(u8).to(DEV)
    params, feat = eng.forward(x, want_pool=True)
    lmk, p2 = eng.forward_landmarks(x, want_params=True)
    lmk_u8, p3 = eng.forward_landmarks(u8.to(DEV), want_params=True)
    assert torch.equal(_i32(p2), _i32(params)) and torch.equal(_i32(p3), _i32(params))
    assert torch.equal(_i32(lmk_u8), _i32(lmk))
    return params, feat, lmk


def pool_ratios(eng, fused: bool, sd, x: torch.Tensor) -> Ratios:
    """Every stage of every pool face against block64, ORACLE_CHUNK faces at a time."""
    total = Ratios()
    for f0 in range(0, P, ORACLE_CHUNK):
        faces = list(range(f0, min(P, f0 + ORACLE_CHUNK)))
        for s, (r, loc, kind) in stage_ratios(eng, fused, sd, x, faces).items():
            if s not in total or r >= total[s][0]:
                total[s] = (r, (faces[loc[0]],) + tuple(loc[1:]), kind)
    return total


# ---- A. the pool, then every face of every placement batch --------------------------------------------------------------
@pytest.mark.parametrize('engine', list(ENGINES))
def test_every_face_has_its_pool_bits(model, sd, pool_u8, batches, engine):
    fused = engine == 'tc_fused'
    eng = _engine(model, ENGINES[engine])
    try:
        x_pool = synthetic.normalize_crops(pool_u8).to(DEV)
        ratios = pool_ratios(eng, fused, sd, x_pool)
        report(f'{engine} pool P={P}, every face', ratios)
        bad = over(engine, ratios)
        assert not bad, bad
        params, feat, lmk = pool_outputs(eng, pool_u8)
        rows = {bytes(r) for r in _i32(params).cpu().numpy()}
        assert len(rows) == P, 'two pool faces share their params bits'
        if fused:
            blocks = [eng.debug_forward_until(x_pool, 3 * b - 1) for b in range(1, 18)]
        for kind, b in batches.items():
            place = tile_cover.placement(b, P)
            u8 = pool_u8.index_select(0, place).to(DEV)
            x = synthetic.normalize_crops(u8)
            got_p, got_f = eng.forward(x, want_pool=True)
            _assert_same(f'{engine} {kind} B={b} params', got_p, params, place)
            _assert_same(f'{engine} {kind} B={b} pooled feature', got_f, feat, place)
            for name, inp in (('fp32', x), ('uint8', u8)):
                got_l, got_lp = eng.forward_landmarks(inp, want_params=True)
                _assert_same(f'{engine} {kind} B={b} {name} landmarks', got_l, lmk, place)
                _assert_same(f'{engine} {kind} B={b} {name} params', got_lp, params, place)
            if fused:
                for blk in range(1, 18):
                    _assert_same(f'{engine} {kind} B={b} block {blk}', eng.debug_forward_until(x, 3 * blk - 1),
                                 blocks[blk - 1], place)
            elif kind == 'odd_pairs':
                for spec in conv_plan():
                    ref = eng.debug_forward_until(x_pool, spec.index)
                    _assert_same(f'{engine} {kind} B={b} conv {spec.index}', eng.debug_forward_until(x, spec.index),
                                 ref, place)
                    del ref
            if kind == 'bench':
                again_p, again_f = eng.forward(x, want_pool=True)
                assert torch.equal(_i32(again_p), _i32(got_p)) and torch.equal(_i32(again_f), _i32(got_f))
                controls(eng, u8, got_p, params, place)
        assert eng.poll_error() == 0 and eng.poll_saturation(warn=False) == 0
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)


def controls(eng, u8, got_p, params, place):
    """E. One pixel of one face changed by 1: that face alone leaves its pool bits.  The comparison, given the placement
    shifted by one face, reports every face."""
    b = u8.shape[0]
    f = 777
    bumped = u8.clone()
    v = int(bumped[f, 1, 60, 61])
    bumped[f, 1, 60, 61] = v + 1 if v < 255 else v - 1
    p = eng.forward(synthetic.normalize_crops(bumped))
    assert differing_faces(p, params, place) == [f]
    assert differing_faces(got_p, params, (place + 1) % P) == list(range(b))


# ---- B. host pipelines -------------------------------------------------------------------------------------------------------
def _host_batch(pool_u8, b, kind):
    """Batch b of the placement as a host tensor: 'u8' pinned uint8, 'f32' pinned fp32, 'pageable' fp32."""
    place = tile_cover.placement(b, P)
    u8 = pool_u8.index_select(0, place).contiguous()
    x = u8 if kind == 'u8' else synthetic.normalize_crops(u8)
    return (x if kind == 'pageable' else x.pin_memory()), place


def _host_out(b, n_pts):
    return torch.empty((b, 3, n_pts), dtype=torch.float32).pin_memory(), torch.empty((b, 62), dtype=torch.float32).pin_memory()


def test_host_pipelines_every_face(model, pool_u8):
    eng = _engine(model, _lib.ENGINE_TC_FUSED)
    params, _, lmk = pool_outputs(eng, pool_u8)
    n_pts = eng.n_pts
    big = {k: _host_batch(pool_u8, 2100, k) for k in ('f32', 'pageable', 'u8')}
    sub = lambda k, b: (big[k][0][:b], big[k][1][:b])              # the first b faces of a placement are its batch b

    def check(tag, place, lmk_out, par_out=None):
        _assert_same(f'{tag} landmarks', lmk_out, lmk, place)
        if par_out is not None:
            _assert_same(f'{tag} params', par_out, params, place)

    # submit / wait: full 1024-face chunks, a ragged last chunk, a staging slot reused within one call
    for b in (1025, 2100):
        for k in ('f32', 'pageable', 'u8'):
            x, place = sub(k, b)
            lo, po = _host_out(b, n_pts)
            assert eng.host_wait(eng.forward_landmarks_host_submit(x, lo, po)) is lo
            check(f'submit {k} B={b}', place, lo, po)
    # two multi-chunk calls in flight, then a third submit (which waits for the first)
    calls = [('u8', 2100), ('f32', 1025), ('f32', 2100)]
    outs = [_host_out(b, n_pts) for _, b in calls]
    tickets = [eng.forward_landmarks_host_submit(sub(k, b)[0], *outs[i]) for i, (k, b) in enumerate(calls)]
    for i, ((k, b), tk) in enumerate(zip(calls, tickets)):
        assert eng.host_wait(tk) is outs[i][0]
        check(f'in flight {i} {k} B={b}', sub(k, b)[1], *outs[i])

    # the blocking C entries: a 512-face first chunk, then 512-face chunks
    lib, h = eng._lib, eng._h
    torch.cuda.synchronize()

    def blocking(k, b, with_params):
        x, place = sub('u8' if k == 'u8' else 'f32', b)
        lo, po = _host_out(b, n_pts)
        fn = lib.syn_forward_landmarks_host_u8 if k == 'u8' else lib.syn_forward_landmarks_host
        _lib.check(fn(h, x.data_ptr(), b, po.data_ptr() if with_params else None, lo.data_ptr()))
        check(f'blocking {k} B={b} params={with_params}', place, lo, po if with_params else None)

    for b in (1, 511, 512, 513, 1100):
        for k in ('f32', 'u8'):
            for with_params in (False, True):
                blocking(k, b, with_params)
    # blocking calls between submitted ones on the same handle: chunk sizes and staging-slot parity alternate
    first = [('u8', 1100), ('f32', 2100)]
    outs = [_host_out(b, n_pts) for _, b in first]
    t0 = eng.forward_landmarks_host_submit(sub(*first[0])[0], *outs[0])
    blocking('f32', 513, True)
    t1 = eng.forward_landmarks_host_submit(sub(*first[1])[0], *outs[1])
    blocking('u8', 1100, False)
    blocking('u8', 1, True)
    for i, tk in enumerate((t0, t1)):
        assert eng.host_wait(tk) is outs[i][0]
        check(f'interleaved {first[i]}', sub(*first[i])[1], *outs[i])
    assert eng.poll_error() == 0 and eng.poll_saturation(warn=False) == 0


@pytest.mark.parametrize('engine', ['simt_fp32', 'tc_bf16x3'])
def test_unfused_engines_host_uint8_every_face(model, pool_u8, engine):
    """The unfused engines normalise uint8 crops into a scratch buffer first (d_x_f32), sized by the chunk."""
    eng = _engine(model, ENGINES[engine])
    try:
        params, _, lmk = pool_outputs(eng, pool_u8)
        x, place = _host_batch(pool_u8, 2100, 'u8')
        lo, po = _host_out(2100, eng.n_pts)
        eng.forward_landmarks_host(x, lo, po)
        _assert_same(f'{engine} host uint8 B=2100 landmarks', lo, lmk, place)
        _assert_same(f'{engine} host uint8 B=2100 params', po, params, place)
        assert eng.poll_error() == 0
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)


# ---- C. the centre-crop frame on every uint8 stem ---------------------------------------------------------------------------
MARGINS = (0, 1, 3, 4, 5, 8, 59)


def _frame_check(eng, run, u8, tag, host=None):
    """For every margin: ``run`` on the uint8 crops with the frame set == ``run`` on the host-framed, host-normalised
    fp32 crops; margin 0 restores the unframed bits; -1 and 60 are refused and leave the margin as it was."""
    lib, h = eng._lib, eng._h
    plain = run(synthetic.normalize_crops(u8).to(DEV))
    try:
        for m in MARGINS:
            eng.set_center_crop(m)
            want = run(synthetic.normalize_crops(framed(u8, m)).to(DEV))
            got = run(u8.to(DEV))
            for g, w in zip(got, want):
                assert torch.equal(_i32(g), _i32(w)), f'{tag} margin {m}'
            if m > 0:
                assert not torch.equal(_i32(want[0]), _i32(plain[0])), f'{tag} margin {m} changes nothing'
            if host is not None:
                host(u8, want, m)
        eng.set_center_crop(5)
        five = run(u8.to(DEV))
        for bad in (-1, 60):
            assert lib.syn_set_center_crop(h, bad) == 1                           # SYN_ERR_INVALID
        for g, w in zip(run(u8.to(DEV)), five):
            assert torch.equal(_i32(g), _i32(w)), f'{tag}: a refused margin changed the frame'
        eng.set_center_crop(0)
        for g, w in zip(run(u8.to(DEV)), plain):
            assert torch.equal(_i32(g), _i32(w)), f'{tag}: margin 0 does not restore the unframed bits'
    finally:
        eng.set_center_crop(0)


@pytest.mark.parametrize('engine', list(ENGINES))
def test_center_crop_mobilenet_v2(model, engine):
    """The fused stem (engine 2) and normalize_u8_kernel (engines 0 and 1), through the device and the host entries."""
    eng = _engine(model, ENGINES[engine])
    u8 = synthetic.make_structured_crops_u8(13, seed=515)
    lib, h = eng._lib, eng._h

    def run(x):
        lmk, params = eng.forward_landmarks(x, want_params=True)
        return lmk, params

    def host(u8, want, m):
        lo, po = _host_out(u8.shape[0], eng.n_pts)
        eng.forward_landmarks_host(u8.pin_memory(), lo, po)
        assert torch.equal(_i32(lo), _i32(want[0].cpu())) and torch.equal(_i32(po), _i32(want[1].cpu())), m
        lo2, po2 = _host_out(u8.shape[0], eng.n_pts)
        x = u8.pin_memory()
        torch.cuda.synchronize()
        _lib.check(lib.syn_forward_landmarks_host_u8(h, x.data_ptr(), u8.shape[0], po2.data_ptr(), lo2.data_ptr()))
        assert torch.equal(_i32(lo2), _i32(lo)) and torch.equal(_i32(po2), _i32(po)), m

    try:
        _frame_check(eng, run, u8, engine, host)
        assert eng.poll_error() == 0
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)


@pytest.mark.parametrize('arch', ['resnet18', 'mobilenet_05'])
def test_center_crop_convbn_stems(synth_pack, arch):
    """resnet_stem_kernel and mbv1_stem_kernel, which frame and normalise the uint8 crop while staging it."""
    if arch.startswith('resnet'):
        m = make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
        eng = m._engine(DEV)
        run = eng.forward_resnet
    else:
        m = make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)
        eng = m._engine(DEV)
        run = eng.forward_mobilenet_v1
    _frame_check(eng, run, synthetic.make_structured_crops_u8(13, seed=516), arch)
    assert eng.poll_error() == 0


# ---- D. the detector's frame batch at its limit ------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def fb_sd():
    return synthetic.make_faceboxes_state_dict(0)


def test_forward_batch_of_64_full_size_frames(fb_sd):
    """SYN_FB_MAX_FRAMES distinct 720 x 1080 frames in one call: every frame has the bits of its one-image call."""
    n = _lib.FB_MAX_FRAMES
    base = [synthetic.make_scene_u8(720, 1080, 31 + s) for s in range(8)]
    frames = np.stack([np.roll(base[i % 8], 41 * (i // 8), axis=1) for i in range(n)])
    assert len({f.tobytes() for f in frames}) == n
    net = faceboxes.FaceBoxesNet(fb_sd, DEV)
    try:
        stack = torch.from_numpy(frames).to(DEV)
        loc, conf = net.forward_batch(stack)
        for i in range(n):
            l1, c1 = net.forward(stack[i])
            assert torch.equal(_i32(loc[i]), _i32(l1)) and torch.equal(_i32(conf[i]), _i32(c1)), f'frame {i}'
        torch.cuda.synchronize()
    finally:
        net.close()


def test_detect_batch_of_65_frames(fb_sd):
    """65 frames: one full 64-frame chunk and a one-frame chunk, without lowering the limit."""
    frames = np.stack([synthetic.make_scene_u8(240, 320, 6 + 13 * i) for i in range(_lib.FB_MAX_FRAMES + 1)])
    fb = faceboxes.FaceBoxes(weights=fb_sd, device='cuda:0')
    got = fb.detect_batch(list(frames))
    assert len(got) == 65
    assert sum(len(r) for r in got) > 0
    for i in range(65):
        want = fb(frames[i])
        assert [[float(v) for v in b] for b in got[i]] == [[float(v) for v in b] for b in want], f'frame {i}'
