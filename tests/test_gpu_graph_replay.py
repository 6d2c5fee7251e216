"""CUDA-graph replays of every device entry point, bit for bit against eager calls on the same handle.

Every case follows torch's capture recipe: an eager warm-up call at the captured batch (so no workspace has to grow under
capture), capture on a side stream (``torch.cuda.graph``) into static input and output tensors, then k = 3 replays, each
after new inputs were copied into the static input.  Each replay must carry the bits of an eager call on those inputs on
the same handle, the handle's launch count must not move during a replay (the replay runs the recorded kernels, not the
library), and the sticky error and saturation flags stay clear.

The MobileNetV2 replays are tied to the float64 oracle, not only to eager calls: their inputs are pool faces placed with
``tile_cover.placement`` and rotated by one face per replay, the eager pool run is held to ``block64`` at the tail-pool
and params stages, and every face of every replay must carry the bits of its pool face.  Since every face moves to
another pool face from one replay to the next, a replay that read the capture-time input instead of the current one
differs on every face.  Negative controls, asserted in ``test_mobilenet_v2_controls``: a replay without the input
rotation differs from the rotated eager call on every face, and a replay captured on engine 2 differs from eager
engine 1.

A replay runs kernels whose arguments were fixed at capture: workspace pointers, tile plans, the centre-crop margin.  It
is valid while no call grows that handle's workspace and no commit, ``syn_resnet_select`` or ``syn_mbv1_set_widen``
runs; the caller orders replays against eager calls of the same handle (``s2.wait_stream(s1)`` after a replay on s1).
A call that would grow a workspace under capture, the host pipelines and the detector's frame paths refuse the capture
with SYN_ERR_STATE before they launch anything, so the capture stays valid and ends cleanly.  H100 only.
"""
import pytest
import torch

from oracle import block64, synth_mbv1, synth_model, synth_resnet, tile_cover
from oracle.stage_check import ENGINES, Ratios, make_model, over, report
from synergynet_b200 import _lib, faceboxes, synthetic

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
P = 16                       # pool faces of the MobileNetV2 cases
POOL_SEED = 977
K = 3                        # replays per case


# ---- helpers ---------------------------------------------------------------------------------------------------------
def _tuple(out):
    return tuple(out) if isinstance(out, (tuple, list)) else (out,)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _faces_differing(got: torch.Tensor, want: torch.Tensor):
    g, w = got.contiguous().view(got.shape[0], -1), want.contiguous().view(want.shape[0], -1)
    return (g.view(torch.int32) != w.view(torch.int32)).any(1).nonzero().flatten().tolist()


def _flags_clear(eng):
    torch.cuda.synchronize()
    assert eng.poll_error() == 0
    assert eng.poll_saturation(warn=False) == 0


def replay_case(tag, handle, fn, inputs, check=None):
    """Capture ``fn(*inputs[0])`` after an eager warm-up, then replay it on ``inputs[1..K]``.  Each replay must have the
    bits of the eager ``fn`` on the same inputs and must not touch the library (launch count); ``check(r, outs)`` may
    hold replay r's outputs to more.  Returns the graph, its static inputs and outputs."""
    want0 = [o.clone() for o in _tuple(fn(*inputs[0]))]
    static = [t.clone() for t in inputs[0]]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = _tuple(fn(*static))
    g.replay()                                                  # the capture's own inputs first
    for o, w in zip(outs, want0):
        assert _same(o, w), f'{tag}: replay of the capture inputs'
    for r in range(1, len(inputs)):
        for s, new in zip(static, inputs[r]):
            s.copy_(new)
        n0 = handle.launch_count
        g.replay()
        assert handle.launch_count == n0, f'{tag}: a replay went through the library'
        want = _tuple(fn(*inputs[r]))
        for i, (o, w) in enumerate(zip(outs, want)):
            assert _same(o, w), f'{tag}: replay {r} output {i} differs from the eager call'
        if check is not None:
            check(r, outs)
    torch.cuda.synchronize()
    return g, static, outs


@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def model(synth_pack, sd):
    return make_model(sd)


@pytest.fixture(scope='module')
def pool_u8():
    u8 = synthetic.make_structured_crops_u8(P, seed=POOL_SEED)
    assert len({bytes(f.numpy().tobytes()) for f in u8}) == P
    return u8


@pytest.fixture(scope='module')
def mbv2_batches():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [1, *tile_cover.choose_batches(sms).values(), 1024]


def _engine(model, kind):
    model.set_engine(kind)
    return model._engine(DEV)


def pool_run(eng, fused, sd, pool_u8):
    """The eager pool run at B = P: (params, pooled feature, landmarks), held to block64 at the tail-pool and params."""
    x = synthetic.normalize_crops(pool_u8).to(DEV)
    params, feat = eng.forward(x, want_pool=True)
    lmk, p2 = eng.forward_landmarks(pool_u8.to(DEV), want_params=True)
    assert _same(p2, params)
    last = eng.debug_forward_until(x, 50 if fused else 51).cpu().double()
    pool_want = block64.tail(sd, last) if fused else block64.avgpool(last)
    ratios = Ratios()
    ratios.add('pool', 'pool', feat.cpu().double(), pool_want)
    ratios.add('params', 'params', params.cpu().double(), block64.heads(sd, feat.cpu().double()))
    report(f'engine {eng.engine} replay pool P={P}', ratios)
    name = [k for k, v in ENGINES.items() if v == eng.engine][0]
    assert not over(name, ratios), ratios
    return params, feat, lmk


def _placed(pool_u8, b, r, dtype):
    """Batch b of pool faces, placement rotated by r faces: (input on the device, pool face of every face)."""
    place = (tile_cover.placement(b, P) + r) % P
    u8 = pool_u8.index_select(0, place).to(DEV)
    return (u8 if dtype == 'uint8' else synthetic.normalize_crops(u8)), place


# ---- MobileNetV2: both entries, three engines, fp32 and uint8, B = 1, the tile-cover batches and 1024 -------------------
@pytest.mark.parametrize('engine', list(ENGINES))
def test_mobilenet_v2_replays_carry_pool_bits(model, sd, pool_u8, mbv2_batches, engine):
    fused = engine == 'tc_fused'
    eng = _engine(model, ENGINES[engine])
    try:
        params, feat, lmk = pool_run(eng, fused, sd, pool_u8)
        for b in sorted(mbv2_batches, reverse=True):
            for dtype in ('fp32', 'uint8'):
                ins, places = zip(*[_placed(pool_u8, b, r, dtype) for r in range(K + 1)])
                ins = [(x,) for x in ins]

                def check_lmk(r, outs, places=places, tag=f'{engine} B={b} {dtype} forward_landmarks'):
                    for name, got, pool in (('landmarks', outs[0], lmk), ('params', outs[1], params)):
                        bad = _faces_differing(got, pool.index_select(0, places[r].to(DEV)))
                        assert not bad, f'{tag} replay {r} {name}: faces {bad[:8]} differ from their pool face'

                def check_fwd(r, outs, places=places, tag=f'{engine} B={b} {dtype} forward'):
                    for name, got, pool in (('params', outs[0], params), ('pooled feature', outs[1], feat)):
                        bad = _faces_differing(got, pool.index_select(0, places[r].to(DEV)))
                        assert not bad, f'{tag} replay {r} {name}: faces {bad[:8]} differ from their pool face'

                replay_case(f'{engine} B={b} {dtype} forward_landmarks', eng,
                            lambda x: eng.forward_landmarks(x, want_params=True), ins, check_lmk)
                if dtype == 'fp32':          # forward has no uint8 entry
                    replay_case(f'{engine} B={b} forward', eng, lambda x: eng.forward(x, want_pool=True), ins, check_fwd)
        _flags_clear(eng)
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)


def test_mobilenet_v2_controls(model, pool_u8):
    """Negative controls of the bit comparisons: a replay whose input was not rotated differs from the rotated eager
    call on every face; a replay captured on engine 2 differs from eager engine 1 on the same input."""
    b = 1024
    eng = _engine(model, _lib.ENGINE_TC_FUSED)
    try:
        x0, _ = _placed(pool_u8, b, 0, 'fp32')
        x1, _ = _placed(pool_u8, b, 1, 'fp32')
        g, static, outs = replay_case('control', eng, lambda x: eng.forward_landmarks(x, want_params=True), [(x0,)])
        g.replay()                                           # static input still holds rotation 0
        rotated = eng.forward_landmarks(x1, want_params=True)
        assert _faces_differing(outs[1], rotated[1]) == list(range(b))
        assert _faces_differing(outs[0], rotated[0]) == list(range(b))
        static[0].copy_(x1)
        g.replay()
        assert _same(outs[1], rotated[1])
        eng.set_engine(_lib.ENGINE_TC_BF16X3)
        other = eng.forward_landmarks(x1, want_params=True)
        assert not _same(outs[1], other[1]) and not _same(outs[0], other[0])
        _flags_clear(eng)
    finally:
        model.set_engine(_lib.ENGINE_TC_FUSED)


@pytest.mark.parametrize('engine', ['tc_fused', 'simt_fp32'])
def test_center_crop_margin_is_fixed_at_capture(model, engine):
    """The uint8 stems read the centre-crop margin as a launch argument: a replay keeps the margin set at capture time,
    whatever ``set_center_crop`` set since (documented in include/synergy_b200.h)."""
    eng = _engine(model, ENGINES[engine])
    ins = [(synthetic.make_structured_crops_u8(13, seed=880 + r).to(DEV),) for r in range(K + 1)]
    fn = lambda x: eng.forward_landmarks(x, want_params=True)
    try:
        eng.set_center_crop(5)
        g, static, outs = replay_case(f'{engine} margin 5', eng, fn, ins)
        framed5 = [o.clone() for o in outs]
        eng.set_center_crop(0)
        g.replay()                                           # static input = ins[K]
        plain = fn(ins[K][0])
        assert _same(outs[1], framed5[1]) and _same(outs[0], framed5[0])
        assert not _same(outs[1], plain[1])
        _flags_clear(eng)
    finally:
        eng.set_center_crop(0)
        model.set_engine(_lib.ENGINE_TC_FUSED)


# ---- the conv+BN backbones ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('arch', ['resnet18', 'resnet50', 'mobilenet_05'])
def test_convbn_backbone_replays(synth_pack, arch):
    if arch.startswith('resnet'):
        m = make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
        run = m._engine(DEV).forward_resnet
    else:
        m = make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)
        run = m._engine(DEV).forward_mobilenet_v1
    eng = m._engine(DEV)
    for b in (128, 13):                                      # the tile-edge batches of the GEMM-layer tests
        for dtype in ('fp32', 'uint8'):
            u8 = [synthetic.make_structured_crops_u8(b, seed=300 + 7 * r + b).to(DEV) for r in range(K + 1)]
            ins = [(u if dtype == 'uint8' else synthetic.normalize_crops(u),) for u in u8]
            replay_case(f'{arch} B={b} {dtype}', eng, run, ins)
    _flags_clear(eng)


# ---- PointNet heads and losses -------------------------------------------------------------------------------------------
def test_pointnet_and_loss_replays(model):
    b = 37
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(4, seed=1)).to(DEV)
    eng = model._pointnet_engine(x, 0)
    assert model._pointnet_engine(x, 1) is eng
    gen = torch.Generator().manual_seed(37)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=gen) * scale).to(DEV)
    ins = [(rnd(b, 3, 68, scale=40.0), rnd(b, 1280).abs(), rnd(b, 62), rnd(b, 3, 68, scale=40.0), rnd(b, 62))
           for _ in range(K + 1)]
    replay_case('mlp_for', eng, lambda l, p, q, t, u: eng.mlp_for(l, p, q), ins)
    replay_case('mlp_rev', eng, lambda l, p, q, t, u: eng.mlp_rev(l), ins)
    replay_case('wing_loss', eng, lambda l, p, q, t, u: eng.wing_loss(l, t), ins)
    for mode in ('normal', 'only_3dmm'):
        replay_case(f'param_loss {mode}', eng, lambda l, p, q, t, u: eng.param_loss(q, u, mode=mode), ins)
    _flags_clear(eng)


# ---- reconstruction and pose (the dense case captures the programmatic-dependent launch) ------------------------------
@pytest.mark.parametrize('b', [1, 129])
def test_reconstruction_and_pose_replays(model, b):
    eng = _engine(model, _lib.ENGINE_TC_FUSED)
    params = [eng.forward(synthetic.normalize_crops(synthetic.make_structured_crops_u8(b, seed=500 + r)).to(DEV))
              for r in range(K + 1)]
    gen = torch.Generator().manual_seed(b)
    roi5 = (torch.rand(b, 5, generator=gen) * torch.tensor([3.0, 400.0, 3.0, 300.0, 3.0]) + 0.5).to(DEV)
    ins = [(p,) for p in params]
    for dense in (False, True):
        replay_case(f'reconstruct B={b} dense={dense}', eng, lambda p: eng.reconstruct(p, dense=dense), ins)
        replay_case(f'reconstruct_image B={b} dense={dense}', eng, lambda p: eng.reconstruct_image(p, roi5, dense=dense), ins)
    replay_case(f'pose_decode B={b}', eng, lambda p: eng.pose_decode(p, roi5), ins)
    replay_case(f'pose_decode B={b} no roi', eng, lambda p: eng.pose_decode(p), ins)
    _flags_clear(eng)


# ---- the detector network: the one-image path ------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def fb_sd():
    return synthetic.make_faceboxes_state_dict(0)


def test_detector_one_image_replays(fb_sd):
    net = faceboxes.FaceBoxesNet(fb_sd, DEV)
    try:
        for h, w in ((720, 1080), (1, 1)):
            if h == 1:
                ins = [(torch.full((1, 1, 3), 17 * r + 3, dtype=torch.uint8, device=DEV),) for r in range(K + 1)]
            else:
                ins = [(torch.from_numpy(synthetic.make_scene_u8(h, w, 60 + r)).to(DEV),) for r in range(K + 1)]
            replay_case(f'detector {h}x{w}', net, net.forward, ins)
    finally:
        torch.cuda.synchronize()
        net.close()


# ---- a replay ordered before an eager call on another stream ----------------------------------------------------------------
def test_replay_then_eager_on_another_stream(model, pool_u8):
    """Replay on s1, ``s2.wait_stream(s1)``, then an eager call on s2: both results are the eager-only ones.  Without
    the wait the two share the workspace unordered: a data race by construction, not tested."""
    eng = _engine(model, _lib.ENGINE_TC_FUSED)
    b = 1024
    xs = [_placed(pool_u8, b, r, 'fp32')[0] for r in range(3)]
    fn = lambda x: eng.forward_landmarks(x, want_params=True)
    want = [[o.clone() for o in fn(x)] for x in xs]
    g, static, outs = replay_case('ordering', eng, fn, [(xs[0],)])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        static[0].copy_(xs[1])
        g.replay()
    s2.wait_stream(s1)
    with torch.cuda.stream(s2):
        eager = fn(xs[2])
    torch.cuda.synchronize()
    assert _same(outs[0], want[1][0]) and _same(outs[1], want[1][1])
    assert _same(eager[0], want[2][0]) and _same(eager[1], want[2][1])
    _flags_clear(eng)


# ---- refusals: a capture that would grow a workspace, the host pipelines, the detector's frame paths --------------------------
def refused(tag, call, *patterns):
    """Run ``call`` under capture on a side stream after a marker op: it must raise SYN_ERR_STATE naming ``patterns``,
    and the capture must still be valid -- it ends cleanly and its replay runs the marker."""
    marker = torch.zeros(1, device=DEV)
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        marker.add_(1)
        with pytest.raises(_lib.SynergyLibError) as ei:
            call()
    assert ei.value.code == _lib.SYN_ERR_STATE, f'{tag}: {ei.value}'
    msg = str(ei.value)
    for p in patterns:
        assert p in msg, f'{tag}: {p!r} not in {msg!r}'
    g.replay()
    torch.cuda.synchronize()
    assert marker.item() == 1.0, f'{tag}: the capture did not survive the refusal'
    del g


GROW = 'eager call before capture'


def test_refused_growth_mobilenet_v2(synth_pack, sd):
    """ensure_workspace, the uint8 crops' fp32 scratch and the reconstruction tiles."""
    m = make_model(sd)
    eng = _engine(m, _lib.ENGINE_SIMT_FP32)
    u8 = {b: synthetic.make_structured_crops_u8(b, seed=b).to(DEV) for b in (4, 8)}
    x = {b: synthetic.normalize_crops(u) for b, u in u8.items()}
    before = [o.clone() for o in eng.forward(x[4], want_pool=True)]
    refused('activation workspace', lambda: eng.forward(x[8]), 'batch 8', 'activation workspace', GROW)
    params8 = eng.forward(x[8])                              # the workspace now holds 8 faces, the tiles and scratch none
    eng.set_engine(_lib.ENGINE_TC_FUSED)
    refused('reconstruction tiles', lambda: eng.reconstruct(params8), 'batch 8', 'reconstruction tiles', GROW)
    # forward_landmarks grows every buffer before its first launch: the refused call records no backbone launch
    refused('forward_landmarks tiles', lambda: eng.forward_landmarks(x[8]), 'batch 8', 'reconstruction tiles', GROW)
    eng.forward_landmarks(x[8])
    eng.set_engine(_lib.ENGINE_SIMT_FP32)
    refused('fp32 scratch', lambda: eng.forward_landmarks(u8[8]), 'batch 8', 'fp32 scratch', GROW)
    after = eng.forward(x[4], want_pool=True)
    assert all(_same(a, b) for a, b in zip(after, before))
    eng.forward_landmarks(u8[8])
    _flags_clear(eng)


def test_refused_growth_convbn_and_pointnet(synth_pack):
    m = make_model(synth_resnet.build_resnet_state_dict(0, 'resnet18'), 'resnet18', strict=False)
    eng = m._engine(DEV)
    x = {b: synthetic.normalize_crops(synthetic.make_structured_crops_u8(b, seed=b)).to(DEV) for b in (4, 8)}
    before = [o.clone() for o in eng.forward_resnet(x[4])]
    refused('backbone workspace', lambda: eng.forward_resnet(x[8]), 'batch 8', 'backbone workspace', GROW)
    assert all(_same(a, b) for a, b in zip(eng.forward_resnet(x[4]), before))
    _flags_clear(eng)

    lmk = {b: torch.randn(b, 3, 68, generator=torch.Generator().manual_seed(b)).to(DEV) * 40 for b in (4, 8)}
    fresh = make_model(synth_model.build_state_dict(0))
    heads = fresh._pointnet_engine(x[4], 1)
    before = heads.mlp_rev(lmk[4]).clone()
    refused('PointNet workspace', lambda: heads.mlp_rev(lmk[8]), 'batch 8', 'PointNet workspace', GROW)
    assert _same(heads.mlp_rev(lmk[4]), before)
    _flags_clear(heads)


def test_refused_host_pipelines(model):
    eng = _engine(model, _lib.ENGINE_TC_FUSED)
    x = synthetic.make_structured_crops_u8(4, seed=3).pin_memory()
    before = eng.forward_landmarks_host(x).clone()
    refused('host', lambda: eng.forward_landmarks_host(x), 'batch 4', 'cannot be captured')
    refused('host submit', lambda: eng.forward_landmarks_host_submit(x), 'batch 4', 'cannot be captured')
    assert _same(eng.forward_landmarks_host(x), before)
    _flags_clear(eng)


def test_refused_detector(fb_sd):
    net = faceboxes.FaceBoxesNet(fb_sd, DEV)
    try:
        small = torch.from_numpy(synthetic.make_scene_u8(64, 96, 5)).to(DEV)
        big = torch.from_numpy(synthetic.make_scene_u8(720, 1080, 6)).to(DEV)
        before = [o.clone() for o in net.forward(small)]
        refused('detector workspace', lambda: net.forward(big), '720x1080', 'detector workspace', GROW)
        net.forward(big)
        stack = torch.stack([small, small])
        refused('forward_batch', lambda: net.forward_batch(stack), '2 frames', 'cannot be captured')
        refused('forward_images', lambda: net.forward_images([small, big]), '2 frames', 'cannot be captured')
        assert all(_same(a, b) for a, b in zip(net.forward(small), before))
        loc, conf = net.forward_batch(stack)
        assert _same(loc[1], before[0]) and _same(conf[1], before[1])
    finally:
        torch.cuda.synchronize()
        net.close()
