"""Two host threads, each on its own CUDA stream, sharing one library handle: every result equals the single-threaded one.

The handles are not re-entrant and their calls share one activation workspace.  ``Engine`` and ``FaceBoxesNet`` hold a
lock around every call and make a call on another stream wait for the previous call's device work
(``engine.StreamOrder``).  Without that, two threads sharing a ``FaceBoxes`` interleave their launches over one
workspace, and a growth (one thread's images are larger than the other's) frees buffers the other thread's queued kernels
still read.  H100 only.
"""
import threading

import numpy as np
import pytest
import torch

from oracle import synth_mbv1, synth_model, synth_resnet
from oracle.stage_check import make_model
from synergynet_b200 import faceboxes, synthetic

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
ITERS = 8


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and torch.equal(a.contiguous().reshape(-1).view(torch.uint8),
                                              b.contiguous().reshape(-1).view(torch.uint8))


def run_threads(work):
    """``work(t, i)`` for t in 0, 1 on two host threads, each inside its own stream, ITERS times: results[t][i]."""
    got = [[None] * ITERS for _ in range(2)]
    errors = []

    def worker(t):
        try:
            torch.cuda.set_device(0)
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for i in range(ITERS):
                    got[t][i] = work(t, i)
            st.synchronize()
        except BaseException as e:            # re-raised on the main thread
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    torch.cuda.synchronize()
    if errors:
        raise errors[0]
    return got


# ---- the detector ---------------------------------------------------------------------------------------------------------
# thread 1's sizes exceed thread 0's, so the shared workspace grows while thread 0's calls are queued
SIZES = [[(240, 320), (97, 61), (1, 1)], [(720, 1080), (600, 900), (1100, 1500)]]


def _boxes(rects):
    return [[float(v) for v in b] for b in rects]


@pytest.fixture(scope='module')
def fb_sd():
    return synthetic.make_faceboxes_state_dict(0)


@pytest.fixture(scope='module')
def scenes():
    return [[synthetic.make_scene_u8(h, w, 70 + 11 * t + j) for j, (h, w) in enumerate(SIZES[t])] for t in range(2)]


def test_detector_shared_across_threads_and_streams(fb_sd, scenes):
    fb = faceboxes.FaceBoxes(weights=fb_sd, device='cuda:0')
    stacks = [torch.from_numpy(np.stack([scenes[0][0]] * 3)).to(DEV), torch.from_numpy(np.stack([scenes[1][1]] * 3)).to(DEV)]

    def work(t, i):
        one = scenes[t][i % len(scenes[t])]
        loc, conf = fb.net.forward_batch(stacks[t])
        return _boxes_list([fb(one)]), _boxes_list(fb.detect_images(scenes[t])), loc.clone(), conf.clone()

    want = {(t, j): work(t, j) for t in range(2) for j in range(len(scenes[t]))}
    torch.cuda.synchronize()
    # a fresh detector, so that the concurrent run grows the workspace itself
    fb = faceboxes.FaceBoxes(weights=fb_sd, device='cuda:0')
    got = run_threads(work)
    for t in range(2):
        for i in range(ITERS):
            w, g = want[(t, i % len(scenes[t]))], got[t][i]
            assert g[0] == w[0] and g[1] == w[1], f'thread {t} iteration {i}: boxes differ'
            assert _same(g[2], w[2]) and _same(g[3], w[3]), f'thread {t} iteration {i}: forward_batch differs'
    fb.net.close()


def _boxes_list(lists):
    return [_boxes(r) for r in lists]


def test_get_all_outputs_images_shared_detector(synth_pack, fb_sd, scenes):
    model = make_model(synth_model.build_state_dict(0))
    fb = faceboxes.FaceBoxes(weights=fb_sd, device='cuda:0')
    model.face_detector = fb
    try:
        def work(t, i):
            out = model.get_all_outputs_images(scenes[t])
            return [(np.stack(l) if l else None, np.stack(m) if m else None, p) for l, m, p in out]

        want = [work(t, 0) for t in range(2)]
        assert sum(len(p) for w in want for _, _, p in w) > 0, 'no face detected: the comparison would be empty'
        model.face_detector = fb = faceboxes.FaceBoxes(weights=fb_sd, device='cuda:0')
        got = run_threads(work)
        for t in range(2):
            for i in range(ITERS):
                for j, ((gl, gm, gp), (wl, wm, wp)) in enumerate(zip(got[t][i], want[t])):
                    assert (gl is None) == (wl is None) and (gl is None or np.array_equal(gl, wl)), (t, i, j)
                    assert (gm is None) == (wm is None) and (gm is None or np.array_equal(gm, wm)), (t, i, j)
                    assert len(gp) == len(wp) and all(a[0] == b[0] and np.array_equal(a[1], b[1]) for a, b in zip(gp, wp)), (t, i, j)
    finally:
        model.face_detector = None
    eng = model._engine(DEV)
    assert eng.poll_error() == 0


# ---- the engine: the conv+BN backbones, the PointNet head and the dense reconstruction ----------------------------------------
@pytest.mark.parametrize('arch', ['resnet18', 'mobilenet_05'])
def test_convbn_backbones_across_threads_and_streams(synth_pack, arch):
    if arch.startswith('resnet'):
        m = make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False)
        run = m._engine(DEV).forward_resnet
    else:
        m = make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)
        run = m._engine(DEV).forward_mobilenet_v1
    # thread 1's batch is the larger: its first call grows the backbone workspace
    xs = [synthetic.normalize_crops(synthetic.make_structured_crops_u8(b, seed=90 + b)).to(DEV) for b in (16, 96)]
    want = [[o.clone() for o in run(x)] for x in xs]
    m2 = make_model(synth_resnet.build_resnet_state_dict(0, arch), arch, strict=False) if arch.startswith('resnet') else \
        make_model(synth_mbv1.build_mobilenet_v1_state_dict(0, arch), arch, strict=False)
    run2 = m2._engine(DEV).forward_resnet if arch.startswith('resnet') else m2._engine(DEV).forward_mobilenet_v1
    got = run_threads(lambda t, i: [o.clone() for o in run2(xs[t])])
    for t in range(2):
        for i in range(ITERS):
            assert all(_same(g, w) for g, w in zip(got[t][i], want[t])), f'{arch} thread {t} iteration {i}'
    assert m2._engine(DEV).poll_error() == 0


def test_pointnet_and_dense_reconstruction_across_threads_and_streams(synth_pack):
    sd = synth_model.build_state_dict(0)
    gen = torch.Generator().manual_seed(5)
    ins = []
    for b in (8, 40):
        lmk = (torch.randn(b, 3, 68, generator=gen) * 40).to(DEV)
        ins.append((lmk, torch.randn(b, 1280, generator=gen).abs().to(DEV), torch.randn(b, 62, generator=gen).to(DEV) * 0.1))

    def calls(model):
        eng = model._pointnet_engine(ins[0][0], 0)

        def work(t, i):
            lmk, pool, params = ins[t]
            res, ref = eng.mlp_for(lmk, pool, params)
            return [res.clone(), ref.clone(), eng.reconstruct(params, dense=True).clone()]
        return eng, work

    _, work = calls(make_model(sd))
    want = [work(t, 0) for t in range(2)]
    eng, work = calls(make_model(sd))                       # a fresh handle: the threads grow its workspaces
    got = run_threads(work)
    for t in range(2):
        for i in range(ITERS):
            assert all(_same(g, w) for g, w in zip(got[t][i], want[t])), f'thread {t} iteration {i}'
    assert eng.poll_error() == 0
