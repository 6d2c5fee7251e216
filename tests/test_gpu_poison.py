"""Every device entry on stale and on poisoned workspaces and outputs, bit for bit against a clean call.

The other GPU tests run on memory that already looks valid.  A handle's workspaces only grow and are never cleared, so a
call made after a larger one runs on that call's finite, plausible bytes past its own batch; and the wrappers allocate
their outputs and workspaces with ``torch.empty``, which the caching allocator often serves from a block an earlier call
used.  A kernel that reads a row past the batch, skips a write to its output or relies on a buffer it never cleared can
then pass unnoticed.

Every test follows one protocol over its cases (``check_cases``):

1. a clean call on the inputs of every case gives R0;
2. a larger call with other inputs leaves valid-looking stale bytes past every case's extent in every workspace, and
   frees Python-side buffers (candidate lists, masks, keys, boxes, ...) that later allocations are served from;
3. stale: every case again, with no fill and the plain ``torch.empty``, must return the bits of R0.  This is the pass
   that exercises the index-bearing buffers: a count, key image or box list whose clear were missing would start from an
   earlier call's values;
4. poison: for each of two bytes, ``debug_fill_workspaces(byte)`` sets every byte of every grown workspace of the handle,
   at its allocated size, to ``byte``; every floating-point and uint8 tensor that ``torch.empty`` / ``empty_like`` /
   ``empty_strided`` return during the call is filled the same way (``poisoned_empty``), pinned host outputs are passed
   in pre-filled, and every case must again return the bits of R0.

An output element counts as written when it equals R0 under two different fills (this holds for uint8 images too,
where 0xFF is a legal pixel).  After every stale and poisoned call the sticky error and saturation flags must read 0: a
padded row that reached a clamp holding a stale huge value or NaN would raise a false saturation flag.

Fills.  Float and activation buffers take 0xFF (NaN in every float) and 0x7F (3.4e38, far past the 937.5 clamp of the
split-fp16 engines).  Integer tensors of the poison passes -- counts, candidate and keep lists, NMS masks, key images,
mesh boxes and key offsets -- are cleared to 0x00, and ``syn_fb_debug_fill_workspaces`` clears the detector's geometry
table, so that a byte pattern can never become an out-of-range address; those buffers are exercised by the stale pass.
The exceptions are outputs no kernel of the call reads: the decode's and NMS's counts are pre-set to -1 in every pass, so
a count left unwritten (an empty frame's included) reads -1.  Where each index-bearing value read in a call is written
earlier in the same call:

* decode: the candidate count of every frame is cleared by a memset in ``syn_faceboxes_decode*`` before
  ``faceboxes_select_kernel`` appends to it; ``faceboxes_rank_decode_kernel`` reads only the first ``count`` indices
  and writes ``n_dets`` without reading it;
* NMS: ``nms_mask_kernel`` writes every mask word of every row below the frame's count before ``nms_scan_kernel`` reads
  them in the next launch; the scan writes the keep list and the count without reading either;
* Sim3DR: the key image is cleared by a memset before ``raster_depth_kernel``; the mesh boxes are set to 0x7F7F7F7F by a
  memset before ``mesh_box_kernel`` narrows them; ``mesh_box_scan_kernel`` writes every key offset before
  ``raster_resolve_frames_kernel`` reads them; the extent statistics of the lighting pass (float bit patterns, not
  indices, so they take the float fills) are cleared by a memset before ``mesh_extent_kernel``;
* detector: the frame paths copy their geometry table from the host before the first launch that reads it; the
  one-image path never reads it;
* crops: the plans are built on the host and uploaded whole from a numpy buffer, never from ``torch.empty``.

What this file cannot see: allocations that do not go through those three Python names (``torch.zeros`` / ``full``,
numpy uploads, the library's own ``cudaMalloc``) are never poisoned, and the stale pass only sees what the caching
allocator happens to hand back.

The fills themselves are checked: ``bytes_filled`` must equal the sizes the buffer geometry implies for the largest call
seen so far, for every kind of buffer a handle grows.  ``debug_fill_on_grow`` poisons the buffers a growing call
allocates for itself, and a fill is refused under graph capture.  H100 only.
"""
import contextlib
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import fb64, synth_mbv1, synth_model, synth_resnet, tile_cover
from oracle.stage_check import make_model
from synergynet_b200 import Sim3DR, _lib, detect, faceboxes, inference, synthetic

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
FILLS = (0xFF, 0x7F)
POOL = 64                    # distinct synthetic crops every batch is drawn from

# bytes per face of the MobileNetV2 handle's buffers (synergy_b200.cu, kernels_dense.cuh)
MBV2_WS_PER_FACE = 4 * (2 * 60 * 60 * 32 + 60 * 60 * 96 + 30 * 30 * 144 + 62 + 1280)
RECON_TILE = 64 * 64 * 2 * 2 + 64 * 20 * 4          # per 64-face tile: alpha hi|lo image + pose rows
X_FACE = 3 * 120 * 120
FB_GEO_BYTES = 5 * 4 * 10 * 64                      # FbLevel (5 int32) x 10 levels x SYN_FB_MAX_FRAMES


# ---- helpers ---------------------------------------------------------------------------------------------------------
def _tuple(out):
    return tuple(out) if isinstance(out, (tuple, list)) else (out,)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


def _same(a, b) -> bool:
    if isinstance(a, torch.Tensor):
        return a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bits(a).cpu(), _bits(b).cpu())
    return a == b


def _snap(out):
    return tuple(o.clone() if isinstance(o, torch.Tensor) else o for o in _tuple(out))


def _fill_storage(t: torch.Tensor, byte: int) -> torch.Tensor:
    if t.numel():
        t.untyped_storage().fill_(byte)
    return t


@contextlib.contextmanager
def poisoned_empty(byte: int, int_byte: int = 0):
    """Every tensor ``torch.empty`` / ``empty_like`` / ``empty_strided`` returns is filled with ``byte`` (floating-point,
    uint8) or ``int_byte`` (integer and bool dtypes: counts, indices, keys), on the device and on the host."""
    orig = {n: getattr(torch, n) for n in ('empty', 'empty_like', 'empty_strided')}

    def wrap(fn):
        def poisoned(*args, **kwargs):
            t = fn(*args, **kwargs)
            return _fill_storage(t, byte if t.dtype.is_floating_point or t.dtype == torch.uint8 else int_byte)
        return poisoned

    with pytest.MonkeyPatch.context() as mp:
        for name, fn in orig.items():
            mp.setattr(torch, name, wrap(fn))
        yield


def _flags_clear(eng, tag):
    torch.cuda.synchronize()
    assert eng.poll_error() == 0, f'{tag}: error flag raised'
    assert eng.poll_saturation(warn=False) == 0, f'{tag}: saturation flag raised on an in-range call'


def _expect(tag, got, want, engines):
    torch.cuda.synchronize()
    assert len(got) == len(want), tag
    for i, (g, w) in enumerate(zip(got, want)):
        assert _same(g, w), f'{tag}: output {i} differs from the clean call'
    for e in engines:
        _flags_clear(e, tag)


def check_cases(cases, r0, fill=(), engines=(), int_byte=0):
    """Steps 3 and 4 of the protocol, right after the larger call: every case of ``cases`` ({name: fn}) once stale, then
    every case under each byte of FILLS (the workspaces of every handle in ``fill`` filled first).  Each must return
    ``r0[name]``; ``int_byte=None`` gives integer tensors the float byte too (for integer buffers that hold no index)."""
    for name, fn in cases.items():
        _expect(f'{name} stale', _snap(fn()), r0[name], engines)
    for name, fn in cases.items():
        for byte in FILLS:
            for h in fill:
                h.debug_fill_workspaces(byte)
            with poisoned_empty(byte, byte if int_byte is None else int_byte):
                got = _snap(fn())
            _expect(f'{name} fill 0x{byte:02X}', got, r0[name], engines)


@functools.lru_cache(maxsize=None)
def _pool() -> torch.Tensor:
    return synthetic.make_structured_crops_u8(POOL, seed=977)


def _crops(b, seed):
    """b uint8 crops drawn from the pool of distinct faces, a different draw per seed."""
    g = torch.Generator().manual_seed(seed)
    return _pool().index_select(0, torch.randint(0, POOL, (b,), generator=g))


@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def fb_sd():
    return synthetic.make_faceboxes_state_dict(0)


def _fresh(sd, engine=_lib.ENGINE_TC_FUSED):
    """A new model (so a new library handle, with nothing grown) on ``engine``; needs the ``synth_pack`` fixture."""
    m = make_model(sd)
    m.set_engine(engine)
    return m, m._engine(DEV)


# ---- the fills are real ------------------------------------------------------------------------------------------------
def test_fill_sizes_follow_the_largest_call(synth_pack, sd, fb_sd):
    """Every kind of buffer a handle grows is filled at its allocated size: the MobileNetV2 activations, the
    reconstruction tiles, the uint8 crops' fp32 scratch, the host pipelines' staging, the PointNet workspace, a conv+BN
    backbone workspace and the detector's."""
    m, eng = _fresh(sd)
    assert eng.debug_fill_workspaces(0xFF) == 0                       # nothing grown yet
    x5 = synthetic.normalize_crops(_crops(5, 1)).to(DEV)
    eng.forward(x5)
    total = 5 * MBV2_WS_PER_FACE
    assert eng.debug_fill_workspaces(0xFF) == total
    eng.forward_landmarks(x5)
    total += RECON_TILE
    assert eng.debug_fill_workspaces(0x7F) == total
    eng.forward_landmarks(synthetic.normalize_crops(_crops(3, 2)).to(DEV))   # smaller: nothing grows
    assert eng.debug_fill_workspaces(0x00) == total
    eng.forward_landmarks(synthetic.normalize_crops(_crops(65, 3)).to(DEV))
    total = 65 * MBV2_WS_PER_FACE + 2 * RECON_TILE
    assert eng.debug_fill_workspaces(0x00) == total
    # host pipeline, uint8, blocking, 100 faces: one 100-face chunk -> staging for 100 faces of landmarks and params
    eng.forward_landmarks_host(_crops(100, 4).pin_memory())
    total = 100 * MBV2_WS_PER_FACE + 2 * RECON_TILE + 2 * 100 * X_FACE + 100 * 4 * (3 * eng.n_pts + 62)
    assert eng.debug_fill_workspaces(0xFF) == total
    eng.forward_landmarks_host(synthetic.normalize_crops(_crops(20, 5)).pin_memory())   # fp32 input staging
    total += 2 * 20 * X_FACE * 4
    assert eng.debug_fill_workspaces(0xFF) == total
    # PointNet workspace at 3 faces (M = 204 point rows)
    heads = m._pointnet_engine(x5, 1)
    assert heads is eng
    heads.mlp_rev(torch.randn(3, 3, 68).to(DEV) * 40)
    B, M = 3, 3 * 68
    total += 4 * (2 * M * 512 + M * 64 + B * 2360 + B * 512 + 3 * M + B + B * 1024)
    assert eng.debug_fill_workspaces(0x7F) == total
    _flags_clear(eng, 'fill sizes')

    m0, e0 = _fresh(sd, _lib.ENGINE_SIMT_FP32)                        # engine 0 normalises uint8 crops into a scratch
    e0.forward_landmarks(_crops(5, 6).to(DEV))
    assert e0.debug_fill_workspaces(0xFF) == 5 * MBV2_WS_PER_FACE + RECON_TILE + 5 * X_FACE * 4

    arch, code = 'mobilenet_05', 50                                   # Workspace::fill, shared by the conv+BN backbones
    mb = make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)._engine(DEV)
    base = mb.debug_fill_workspaces(0)
    mb.forward_mobilenet_v1(synthetic.normalize_crops(_crops(7, 7)).to(DEV))
    lib, io, dw = _lib.load(), 0, 0
    for i in range(27):
        d = _lib.ConvDesc()
        _lib.check(lib.syn_mbv1_conv_desc(code, i, C.byref(d)))
        if i % 2:
            dw = max(dw, d.h_out * d.h_out * d.cout)
        else:
            io = max(io, d.h_out * d.h_out * d.cout)
    assert mb.debug_fill_workspaces(0xFF) - base == 7 * 4 * (io + dw + d.cout + 3600 + 16 + 1)

    net = faceboxes.FaceBoxesNet(fb_sd, DEV)
    try:
        assert net.debug_fill_workspaces(0xFF) == 0
        h, w = 200, 300
        net.forward(torch.from_numpy(synthetic.make_scene_u8(h, w, 1)).to(DEV))
        g = {}
        c = lambda n, k, s, p: (n + 2 * p - k) // s + 1
        g[1] = (c(h, 7, 4, 3), c(w, 7, 4, 3))
        g[2] = (c(g[1][0], 3, 2, 1), c(g[1][1], 3, 2, 1))
        g[3] = (c(g[2][0], 5, 2, 2), c(g[2][1], 5, 2, 2))
        for lv in (4, 5, 6):
            g[lv] = (c(g[lv - 1][0], 3, 2, 1), c(g[lv - 1][1], 3, 2, 1))
        pix = {lv: a * b for lv, (a, b) in g.items()}
        floats = [pix[1] * 48, pix[2] * 48, pix[3] * 128] + [pix[4] * n for n in (128, 128, 128, 24, 24, 32, 128)] + \
                 [pix[5] * 256, pix[5] * 128, pix[6] * 256]
        assert net.debug_fill_workspaces(0x7F) == 4 * sum(floats) + FB_GEO_BYTES
    finally:
        torch.cuda.synchronize()
        net.close()


def test_fill_refused_under_capture(synth_pack, sd):
    m, eng = _fresh(sd)
    x = synthetic.normalize_crops(_crops(4, 4)).to(DEV)
    eng.forward(x)
    marker = torch.zeros(1, device=DEV)
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        marker.add_(1)
        with pytest.raises(_lib.SynergyLibError) as ei:
            eng.debug_fill_workspaces(0xFF)
    assert ei.value.code == _lib.SYN_ERR_STATE and 'CUDA graph' in str(ei.value)
    g.replay()
    torch.cuda.synchronize()
    assert marker.item() == 1.0


# ---- MobileNetV2: four engines, fp32 and uint8 crops, a CenterCrop margin, the tile-cover batches after B = 1024 -------
@pytest.fixture(scope='module')
def mbv2_batches():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return sorted([1, *tile_cover.choose_batches(sms).values()])


@pytest.mark.parametrize('engine', [_lib.ENGINE_SIMT_FP32, _lib.ENGINE_TC_BF16X3, _lib.ENGINE_TC_FUSED, _lib.ENGINE_TC_FUSED_1PASS])
def test_mobilenet_v2(synth_pack, sd, mbv2_batches, engine):
    m, eng = _fresh(sd, engine)
    calls = {
        'forward': lambda u8, x: eng.forward(x, want_pool=True),
        'forward_landmarks fp32': lambda u8, x: eng.forward_landmarks(x, want_params=True),
        'forward_landmarks uint8': lambda u8, x: eng.forward_landmarks(u8, want_params=True),
    }
    ins = {b: _crops(b, 100 + b).to(DEV) for b in mbv2_batches}
    ins = {b: (u8, synthetic.normalize_crops(u8)) for b, u8 in ins.items()}
    try:
        for margin in (0, 7):
            eng.set_center_crop(margin)
            run = calls if margin == 0 else {n: fn for n, fn in calls.items() if 'uint8' in n}   # the margin cuts uint8 crops
            cases = {f'engine {engine} margin {margin} B={b} {n}': (lambda fn=fn, b=b: fn(*ins[b]))
                     for b in mbv2_batches for n, fn in run.items()}
            r0 = {n: _snap(fn()) for n, fn in cases.items()}
            big = _crops(1024, 7 + margin).to(DEV)
            for fn in run.values():
                fn(big, synthetic.normalize_crops(big))
            check_cases(cases, r0, [eng], [eng])
    finally:
        eng.set_center_crop(0)


def test_mobilenet_v2_host_pipelines(synth_pack, sd):
    """Blocking calls at 1, 513 and 1100 faces and submitted calls at 1025 and 2100 faces from uint8 crops, and fp32 crops
    at 1 and 1025 faces, into pinned host outputs pre-filled with the poison byte."""
    m, eng = _fresh(sd)
    n_pts = eng.n_pts

    def run(x, submit):                                         # the pinned outputs come from the (poisoned) torch.empty
        b = x.shape[0]
        lmk = torch.empty((b, 3, n_pts), dtype=torch.float32, pin_memory=True)
        par = torch.empty((b, 62), dtype=torch.float32, pin_memory=True)
        if submit:
            eng.host_wait(eng.forward_landmarks_host_submit(x, lmk, par))
        else:
            eng.forward_landmarks_host(x, lmk, par)
        return lmk, par

    keys = [(b, s, 'uint8') for b, s in ((1, False), (513, False), (1100, False), (1025, True), (2100, True))]
    keys += [(1, False, 'fp32'), (1025, True, 'fp32')]
    cases = {}
    for b, s, dt in keys:
        u8 = _crops(b, 200 + b)
        x = (u8 if dt == 'uint8' else synthetic.normalize_crops(u8)).pin_memory()
        cases[f'host pipeline B={b} submit={s} {dt}'] = lambda x=x, s=s: run(x, s)
    r0 = {n: _snap(fn()) for n, fn in cases.items()}
    run(_crops(2300, 9).pin_memory(), True)                   # grows the result staging past every case
    run(synthetic.normalize_crops(_crops(1100, 10)).pin_memory(), True)     # and the fp32 input staging to its full chunk
    check_cases(cases, r0, [eng], [eng])


# ---- the conv+BN backbones -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('arch', ['resnet18', 'resnet50', 'wide_resnet50_2', 'mobilenet_05', 'mobilenet_2'])
def test_convbn_backbones(synth_pack, arch):
    if arch.startswith('mobilenet'):
        m = make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)
        run = m._engine(DEV).forward_mobilenet_v1
    else:
        m = make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
        run = m._engine(DEV).forward_resnet
    eng = m._engine(DEV)
    cases = {}
    for b in (13, 19, 128):
        u8 = _crops(b, 300 + b).to(DEV)
        for dt, x in (('uint8', u8), ('fp32', synthetic.normalize_crops(u8))):
            cases[f'{arch} B={b} {dt}'] = lambda x=x: run(x)
    r0 = {n: _snap(fn()) for n, fn in cases.items()}
    run(synthetic.normalize_crops(_crops(160, 11)).to(DEV))
    check_cases(cases, r0, [eng], [eng])


# ---- PointNet heads and losses --------------------------------------------------------------------------------------------
def test_pointnet_heads_and_losses(synth_pack, sd):
    m, _ = _fresh(sd)
    x = synthetic.normalize_crops(_crops(4, 1)).to(DEV)
    eng = m._pointnet_engine(x, 0)
    assert m._pointnet_engine(x, 1) is eng
    gen = torch.Generator().manual_seed(41)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=gen) * scale).to(DEV)
    ins = {b: (rnd(b, 3, 68, scale=40.0), rnd(b, 1280).abs(), rnd(b, 62), rnd(b, 3, 68, scale=40.0), rnd(b, 62))
           for b in (1, 2, 37, 64)}
    calls = {
        'mlp_for': lambda l, p, q, t, u: eng.mlp_for(l, p, q),
        'mlp_rev': lambda l, p, q, t, u: eng.mlp_rev(l),
        'wing_loss': lambda l, p, q, t, u: eng.wing_loss(l, t),
        'param_loss normal': lambda l, p, q, t, u: eng.param_loss(q, u, mode='normal'),
        'param_loss only_3dmm': lambda l, p, q, t, u: eng.param_loss(q, u, mode='only_3dmm'),
    }
    cases = {f'{n} B={b}': (lambda fn=fn, b=b: fn(*ins[b])) for b in (1, 2, 37) for n, fn in calls.items()}
    r0 = {n: _snap(fn()) for n, fn in cases.items()}
    for fn in calls.values():                                   # the larger call: 64 other faces
        fn(*ins[64])
    check_cases(cases, r0, [eng], [eng])


# ---- reconstruction and pose -----------------------------------------------------------------------------------------------
def test_reconstruction_and_pose(synth_pack, sd):
    m, eng = _fresh(sd)
    base = eng.forward(synthetic.normalize_crops(_crops(129, 5)).to(DEV))
    gen = torch.Generator().manual_seed(4283)

    def params(b, seed):
        g = torch.Generator().manual_seed(seed)
        rep = base.repeat(-(-b // 129), 1)[:b]
        return rep * (1 + 0.01 * torch.randn(rep.shape, generator=g).to(DEV))

    def roi(b):
        return (torch.rand(b, 5, generator=gen) * torch.tensor([3.0, 400.0, 3.0, 300.0, 3.0]) + 0.5).to(DEV)

    sizes = (1, 63, 65, 129)
    ins = {b: (params(b, b), roi(b)) for b in sizes}
    calls = {}
    for dense in (False, True):
        calls[f'reconstruct dense={dense}'] = lambda p, r, d=dense: eng.reconstruct(p, dense=d)
        calls[f'reconstruct dense={dense} unwhitened'] = lambda p, r, d=dense: eng.reconstruct(p, dense=d, whitening=False)
        calls[f'reconstruct_image dense={dense}'] = lambda p, r, d=dense: eng.reconstruct_image(p, r, dense=d)
    calls['pose_decode'] = lambda p, r: eng.pose_decode(p, r)
    calls['pose_decode no roi'] = lambda p, r: eng.pose_decode(p)
    cases = {f'{n} B={b}': (lambda fn=fn, b=b: fn(*ins[b])) for b in sizes for n, fn in calls.items()}
    r0 = {n: _snap(fn()) for n, fn in cases.items()}
    pb, rb = params(4283, 1), roi(4283)
    for fn in calls.values():
        fn(pb, rb)
    del pb, rb
    torch.cuda.empty_cache()
    check_cases(cases, r0, [eng], [eng])


# ---- graph replays after a fill ---------------------------------------------------------------------------------------------
def test_graph_replays_after_a_fill(synth_pack, sd):
    m, eng = _fresh(sd)
    b = 37
    x = synthetic.normalize_crops(_crops(b, 21).to(DEV))
    eng.forward_landmarks(synthetic.normalize_crops(_crops(200, 22)).to(DEV))   # the workspace past the captured batch
    params = eng.forward(x)
    for tag, fn, arg in (('forward_landmarks', lambda t: eng.forward_landmarks(t, want_params=True), x),
                         ('dense reconstruction', lambda t: eng.reconstruct(t, dense=True), params)):
        want = _snap(fn(arg))
        static = arg.clone()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            outs = _tuple(fn(static))
        for byte in FILLS:
            eng.debug_fill_workspaces(byte)
            for o in outs:
                _fill_storage(o, byte)
            g.replay()
            _expect(f'{tag} replay after fill 0x{byte:02X}', outs, want, [eng])
        del g


# ---- growth on poison -----------------------------------------------------------------------------------------------------
def test_growth_on_poison(synth_pack, sd, fb_sd):
    """A call that grows its own workspace, with ``debug_fill_on_grow`` on, returns the clean handle's bits."""
    x = {b: synthetic.normalize_crops(_crops(b, 30 + b)).to(DEV) for b in (3, 70)}
    lmk = {b: torch.randn(b, 3, 68, generator=torch.Generator().manual_seed(b)).to(DEV) * 40 for b in (3, 70)}
    m, clean = _fresh(sd)
    want = {b: _snap(clean.forward_landmarks(x[b], want_params=True)) for b in (3, 70)}
    rev = m._pointnet_engine(x[3], 1)
    want_rev = {b: rev.mlp_rev(lmk[b]).clone() for b in (3, 70)}
    for byte in FILLS:
        m, eng = _fresh(sd)
        eng.debug_fill_on_grow(byte)
        for b in (3, 70):                                         # each call grows every buffer it uses
            _expect(f'MobileNetV2 B={b} grown on 0x{byte:02X}', _snap(eng.forward_landmarks(x[b], want_params=True)), want[b], [])
        heads = m._pointnet_engine(x[3], 1)
        for b in (3, 70):
            _expect(f'mlp_rev B={b} grown on 0x{byte:02X}', (heads.mlp_rev(lmk[b]),), (want_rev[b],), [eng])

    r18 = synth_resnet.build_resnet_state_dict(0, 'resnet18')
    clean = make_model(r18, 'resnet18', strict=False)._engine(DEV)
    want = {b: _snap(clean.forward_resnet(x[b])) for b in (3, 70)}
    for byte in FILLS:
        eng = make_model(r18, 'resnet18', strict=False)._engine(DEV)
        eng.debug_fill_on_grow(byte)
        for b in (3, 70):
            _expect(f'resnet18 B={b} grown on 0x{byte:02X}', _snap(eng.forward_resnet(x[b])), want[b], [eng])

    imgs = [torch.from_numpy(synthetic.make_scene_u8(h, w, 40 + h)).to(DEV) for h, w in ((64, 96), (300, 420))]
    clean = faceboxes.FaceBoxesNet(fb_sd, DEV)
    try:
        want = [_snap(clean.forward(im)) for im in imgs] + [_snap(clean.forward_packed(imgs)[:2])]
        for byte in FILLS:
            net = faceboxes.FaceBoxesNet(fb_sd, DEV)
            try:
                net.debug_fill_on_grow(byte)
                got = [_snap(net.forward(im)) for im in imgs] + [_snap(net.forward_packed(imgs)[:2])]
                for i, (g, w) in enumerate(zip(got, want)):
                    _expect(f'detector call {i} grown on 0x{byte:02X}', g, w, [])
            finally:
                torch.cuda.synchronize()
                net.close()
    finally:
        torch.cuda.synchronize()
        clean.close()


# ---- the detector: network, decode, NMS ---------------------------------------------------------------------------------------
def test_detector_network(fb_sd):
    """The one-image network at the per-stage sizes from largest to smallest, the batched and the image-list paths."""
    sizes = sorted(set(fb64.choose_sizes()), key=lambda s: s[0] * s[1])
    net = faceboxes.FaceBoxesNet(fb_sd, DEV)
    try:
        img = {s: torch.from_numpy(synthetic.make_scene_u8(*s, 50 + i)).to(DEV) for i, s in enumerate(sizes)}
        stack = torch.stack([img[(720, 1080)], torch.zeros_like(img[(720, 1080)])])
        lst = [img[s] for s in sizes[:4]] + [img[sizes[-1]]]
        cases = {f'detector {s}': (lambda s=s: net.forward(img[s])) for s in reversed(sizes)}
        cases['detector batch'] = lambda: net.forward_batch(stack)
        cases['detector images'] = lambda: net.forward_packed(lst)[:2]
        r0 = {n: _snap(fn()) for n, fn in cases.items()}
        net.forward(torch.from_numpy(synthetic.make_scene_u8(1400, 1500, 7)).to(DEV))    # larger than every case
        net.forward_images([torch.from_numpy(synthetic.make_scene_u8(720, 1080, 8 + i)).to(DEV) for i in range(6)])
        check_cases(cases, r0, [net])
    finally:
        torch.cuda.synchronize()
        net.close()


def test_detect_batch_and_images(fb_sd):
    """End to end through the network, decode and NMS of a stack of equal frames and of a list of images of several
    sizes (one above 720 x 1080, shrunk on the device), an all-black frame and a small all-black image among them."""
    fb = faceboxes.FaceBoxes(weights=fb_sd, device=DEV)
    try:
        frames = [synthetic.make_scene_u8(240, 320, 60 + i) for i in range(3)] + [np.zeros((240, 320, 3), np.uint8)]
        images = frames[:2] + [synthetic.make_scene_u8(900, 1300, 64), np.zeros((50, 70, 3), np.uint8)]
        cases = {'detect_batch': lambda: fb.detect_batch(frames), 'detect_images': lambda: fb.detect_images(images)}
        r0 = {n: (fn(),) for n, fn in cases.items()}
        fb.detect_batch([synthetic.make_scene_u8(240, 320, 70 + i) for i in range(9)])
        fb.detect_images([synthetic.make_scene_u8(1000, 1400, 80 + i) for i in range(5)])
        check_cases({n: (lambda fn=fn: (fn(),)) for n, fn in cases.items()}, r0, [fb.net])
    finally:
        torch.cuda.synchronize()
        fb.net.close()


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _counts(n):
    """Count outputs no kernel of the call reads: pre-set to -1, so one left unwritten shows."""
    return torch.full((n,), -1, dtype=torch.int32, device=DEV)


def _decode(loc, conf, hw, scale, top_k):
    """syn_faceboxes_decode on one frame, outputs from ``torch.empty``: (its n rows, n)."""
    p = loc.shape[0]
    cand = torch.empty((p + 1,), dtype=torch.int32, device=DEV)
    dets = torch.empty((top_k, 5), dtype=torch.float32, device=DEV)
    n = _counts(1)
    _lib.check(_lib.load().syn_faceboxes_decode(loc.data_ptr(), conf.data_ptr(), hw[0], hw[1], float(hw[1]), float(hw[0]), scale,
                                                detect.confidence_threshold, top_k, cand.data_ptr(), dets.data_ptr(), n.data_ptr(),
                                                _stream()))
    return dets[:int(n.item())], n


def _decode_frames(loc, conf, hw, scales, top_k, images):
    """syn_faceboxes_decode_batch (images False) or _images on the frames of (N,P,4) / (N,P,2): every frame's n rows, n."""
    nf, p = loc.shape[0], loc.shape[1]
    dets = torch.empty((nf, top_k, 5), dtype=torch.float32, device=DEV)
    n = _counts(nf)
    lib = _lib.load()
    if images:
        cand = torch.empty((nf + nf * p,), dtype=torch.int32, device=DEV)
        hs, ws = np.full(nf, hw[0], np.int32), np.full(nf, hw[1], np.int32)
        sc = np.ascontiguousarray(scales, np.float32)
        _lib.check(lib.syn_faceboxes_decode_images(loc.data_ptr(), conf.data_ptr(), nf, hs.ctypes.data, ws.ctypes.data, sc.ctypes.data,
                                                   detect.confidence_threshold, top_k, cand.data_ptr(), dets.data_ptr(), n.data_ptr(),
                                                   _stream()))
    else:
        cand = torch.empty((nf * (p + 1),), dtype=torch.int32, device=DEV)
        _lib.check(lib.syn_faceboxes_decode_batch(loc.data_ptr(), conf.data_ptr(), nf, hw[0], hw[1], float(hw[1]), float(hw[0]),
                                                  float(scales[0]), detect.confidence_threshold, top_k, cand.data_ptr(),
                                                  dets.data_ptr(), n.data_ptr(), _stream()))
    return [dets[i, :c] for i, c in enumerate(n.tolist())] + [n]


def _nms(dets, n, mode):
    """syn_nms on the first n rows: (the kept indices, their count)."""
    words = (n + 63) // 64
    mask = torch.empty((max(n * words, 1),), dtype=torch.int64, device=DEV)
    keep = torch.empty((max(n, 1),), dtype=torch.int32, device=DEV)
    nk = _counts(1)
    _lib.check(_lib.load().syn_nms(dets.data_ptr(), n, 0.3, mode, mask.data_ptr(), keep.data_ptr(), nk.data_ptr(), _stream()))
    return keep[:int(nk.item())], nk


def _nms_frames(dets, counts, mode):
    """syn_nms_batch: every frame's kept indices, and the counts."""
    nf, rows = dets.shape[0], dets.shape[1]
    mask = torch.empty((nf * rows * ((rows + 63) // 64),), dtype=torch.int64, device=DEV)
    keep = torch.empty((nf, rows), dtype=torch.int32, device=DEV)
    nk = _counts(nf)
    _lib.check(_lib.load().syn_nms_batch(dets.data_ptr(), counts.data_ptr(), nf, rows, 0.3, mode, mask.data_ptr(), keep.data_ptr(),
                                         nk.data_ptr(), _stream()))
    return [keep[i, :k] for i, k in enumerate(nk.tolist())] + [nk]


def _dets(n, seed):
    """n boxes [x1 y1 x2 y2 score] in descending score order, clustered so that NMS suppresses some of them."""
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(n, 2, generator=g) * 200
    xy = torch.where(torch.rand(n, 1, generator=g) < 0.5, xy.round(decimals=-2), xy)
    wh = torch.rand(n, 2, generator=g) * 40 + 10
    score = torch.sort(torch.rand(n, generator=g), descending=True).values
    return torch.cat([xy, xy + wh, score[:, None]], 1).float().contiguous().to(DEV)


CAND_COUNTS = (0, 1, 63, 64, 65)


def _scores(p, count, seed):
    """(p,2) softmax-like scores with exactly ``count`` priors above the threshold (all of them if count is None)."""
    g = torch.Generator().manual_seed(seed)
    face = torch.rand(p, generator=g) * 0.04                  # below confidence_threshold = 0.05
    if count is None:
        face = 0.06 + torch.rand(p, generator=g) * 0.94
    else:
        face[torch.randperm(p, generator=g)[:count]] = 0.06 + torch.rand(count, generator=g) * 0.94
    return torch.stack([1 - face, face], 1)


def test_decode_and_nms():
    """Decode of one frame, a batch and an image list at 0, 1, 63, 64, 65 candidates and above the 5000 cap; NMS at 0, 1,
    63, 64, 65 and 5000 boxes, in one call and per frame.  Rows and keep entries are compared up to their counts (the
    rest is documented unwritten); the counts start at -1 and must be written, an empty frame's included."""
    h, w = 480, 640
    p = detect.num_priors(h, w)
    assert p > 5000
    g = torch.Generator().manual_seed(3)
    counts = list(CAND_COUNTS) + [None]
    loc = (torch.randn(len(counts), p, 4, generator=g) * 0.3).contiguous().to(DEV)
    conf = torch.stack([_scores(p, c, 10 + i) for i, c in enumerate(counts)]).contiguous().to(DEV)
    top_k = detect.top_k
    cases = {f'decode {c} candidates': (lambda i=i: _decode(loc[i], conf[i], (h, w), 1.5, top_k)) for i, c in enumerate(counts)}
    cases['decode_batch'] = lambda: _decode_frames(loc, conf, (h, w), [1.0], top_k, False)
    cases['decode_images'] = lambda: _decode_frames(loc, conf, (h, w), [1.0, 2.0, 0.5, 1.0, 3.0, 0.75], top_k, True)
    big = _dets(5000, 1)
    frames_dets = torch.stack([_dets(65, 10 + i) for i in range(len(CAND_COUNTS))]).contiguous()
    frame_counts = torch.tensor(CAND_COUNTS, dtype=torch.int32, device=DEV)
    for mode in (_lib.NMS_CPU_NMS, _lib.NMS_PY_CPU_NMS):
        for n in CAND_COUNTS + (5000,):
            cases[f'nms mode {mode} n={n}'] = lambda n=n, mode=mode: _nms(big, n, mode)
        cases[f'nms_batch mode {mode}'] = lambda mode=mode: _nms_frames(frames_dets, frame_counts, mode)
    r0 = {n: _snap(fn()) for n, fn in cases.items()}
    want_n = [0, 1, 63, 64, 65, top_k]
    assert [int(r0[f'decode {c} candidates'][1].item()) for c in counts] == want_n
    assert r0['decode_batch'][-1].tolist() == want_n and r0['decode_images'][-1].tolist() == want_n
    assert r0[f'nms_batch mode {_lib.NMS_CPU_NMS}'][-1].tolist()[:2] == [0, 1]
    # the larger calls: every candidate list, mask and keep list holds other values past the cases' extent
    big_conf = torch.stack([_scores(p, None, 90 + i) for i in range(8)]).contiguous().to(DEV)
    big_loc = (torch.randn(8, p, 4, generator=g) * 0.3).contiguous().to(DEV)
    _decode_frames(big_loc, big_conf, (h, w), [1.0] * 8, top_k, True)
    _decode_frames(big_loc, big_conf, (h, w), [1.0], top_k, False)
    _nms(_dets(6000, 2), 6000, _lib.NMS_CPU_NMS)
    _nms_frames(torch.stack([_dets(300, 20 + i) for i in range(8)]).contiguous(),
                torch.full((8,), 300, dtype=torch.int32, device=DEV), _lib.NMS_CPU_NMS)
    check_cases(cases, r0)


# ---- crops ---------------------------------------------------------------------------------------------------------------------
def test_crops():
    img = torch.from_numpy(synthetic.make_scene_u8(300, 400, 90)).to(DEV)
    frames = torch.stack([img, torch.from_numpy(synthetic.make_scene_u8(300, 400, 91)).to(DEV)])
    pack = inference.pack_images([img, torch.from_numpy(synthetic.make_scene_u8(150, 90, 92)).to(DEV)], DEV)
    rois = [[10, 20, 130, 170], [-15, -5, 60, 80], [200, 150, 420, 320]]
    cases = {}
    for mode in (inference.INTER_LINEAR, 4):
        for planar in (True, False):
            cases[f'crop one image mode {mode} planar {planar}'] = \
                lambda m=mode, pl=planar: inference.crop_resize_device(img, rois, (120, 120), m, planar=pl)
            cases[f'crop batch mode {mode} planar {planar}'] = \
                lambda m=mode, pl=planar: inference.crop_resize_frames_device(frames, [0, 1, 1], rois, (120, 120), m, planar=pl)
        cases[f'crop image list mode {mode}'] = \
            lambda m=mode: inference.crop_resize_images_device(pack, [0, 1, 0], rois, [(120, 120), (64, 80), (33, 17)], m)
    r0 = {n: _snap(fn()) for n, fn in cases.items()}
    inference.crop_resize_frames_device(frames, [1] * 40, [[0, 0, 300, 250]] * 40, (120, 120), inference.INTER_LINEAR)
    check_cases(cases, r0)


# ---- Sim3DR and drawing ----------------------------------------------------------------------------------------------------------
def _mesh(seed, b, side=20, h=120, w=160):
    g = torch.Generator().manual_seed(seed)
    ii, jj = torch.meshgrid(torch.arange(side), torch.arange(side), indexing='ij')
    tri = []
    for i in range(side - 1):
        for j in range(side - 1):
            a = i * side + j
            tri += [[a, a + 1, a + side], [a + 1, a + side + 1, a + side]]
    v = torch.stack([jj.flatten().float(), ii.flatten().float(), torch.zeros(side * side)], 1)
    meshes = []
    for _ in range(b):
        s = torch.rand(1, generator=g) * 6 + 2
        off = torch.rand(2, generator=g) * torch.tensor([w * 0.8, h * 0.8]) - 10
        z = torch.randn(side * side, generator=g) * 5
        meshes.append(torch.stack([v[:, 0] * s + off[0], v[:, 1] * s + off[1], z], 1))
    return np.array(tri, np.int32), side * side, torch.stack(meshes).contiguous().to(DEV)


def test_sim3dr_and_drawing():
    tri, nver, verts = _mesh(1, 6)
    _, _, big = _mesh(2, 9)
    r = Sim3DR.MeshRenderer(tri, nver, DEV)
    h, w = 120, 160
    bg = torch.from_numpy(synthetic.make_scene_u8(h, w, 3)).to(DEV)
    frames = torch.stack([bg, bg.flip(0).contiguous(), bg.flip(1).contiguous()])
    counts = [2, 0, 4]
    nrm = r.normals(verts)
    col = r.colors(verts, nrm)
    segs = [[(0, 0, 50, 60, (255, 0, 0)), (10, 100, 150, 5, (0, 255, 0))], [], [(-20, 30, 200, 90, (0, 0, 255))]]
    cases = {
        'Sim3DR normals': lambda: r.normals(verts),
        'Sim3DR rasterize': lambda: r.rasterize(bg.clone(), verts, col, return_depth=True),
        'Sim3DR rasterize_frames': lambda: r.rasterize_frames(frames, verts, col, counts),
        'Sim3DR render_frames': lambda: r.render_frames(frames, verts, counts),
        'add_weighted': lambda: Sim3DR.add_weighted(frames, frames.flip(1).contiguous(), 0.6),
        'draw_lines': lambda: inference.draw_lines_device(frames.clone(), segs),
    }
    colors = {'Sim3DR colors': lambda: r.colors(verts, nrm)}     # its extent statistics take the float fills
    r0 = {n: _snap(fn()) for n, fn in {**cases, **colors}.items()}
    bnrm = r.normals(big)                                       # the larger calls: more meshes, other extents
    bcol = r.colors(big, bnrm)
    r.rasterize(bg.clone(), big, bcol, return_depth=True)
    r.rasterize_frames(torch.cat([frames, frames]), big, bcol, [1, 2, 1, 2, 1, 2])
    check_cases(cases, r0)
    r.colors(big, bnrm)
    check_cases(colors, r0, int_byte=None)
