"""The stem + block-1 kernel (stem_block1_kernel, kernels_stem.cuh) of the fused engines, bit for bit.

The kernel runs two strip pipelines per CTA over a persistent grid, so which CTA, which pipeline and which wave a strip
lands in depends on the batch size and on the face's position in it.  None of that may change a bit of the block-1
output (conv index 2, read through ``Engine.debug_forward_until``):

* every face of batches 1, 2, 3, 131, 132, 133, 265 and 1024 -- uneven pipelines and uneven last waves on a 132-SM
  H100 -- drawn from a pool of crops at random positions, must equal the same crop run alone;
* uint8 crops (normalised and CenterCrop-bordered in the kernel) must give the params and landmarks of the fp32 crops
  with the same values, for border margins 0, 1 and 7;
* a call after a larger one (stale workspaces) and calls on workspaces and outputs poisoned with NaN and 3.4e38 bytes
  must return the clean call's bits and raise neither the saturation nor the error flag.

The float64 check of the block-1 output on a 1024-face batch lives in test_gpu_blocks.py.  H100 only.
"""
import contextlib

import numpy as np
import pytest
import torch

from oracle import synth_model
from oracle.stage_check import make_model, seeded_crops
from synergynet_b200 import synthetic

pytestmark = pytest.mark.gpu

BLOCK1 = 2                                   # conv index 3b - 1 of block 1: the stem kernel's output
BATCHES = (1, 2, 3, 131, 132, 133, 265, 1024)
POOL = 48                                    # distinct crops the batches are drawn from
ENGINES = (2, 3)                             # fused split-fp16 x3, fused single pass


@pytest.fixture(scope='module')
def model(synth_pack):
    return make_model(synth_model.build_state_dict(0))


@pytest.fixture(scope='module')
def pool():
    return seeded_crops(POOL, 517)


def _engine(model, kind):
    model.set_engine(kind)
    return model._engine(torch.device('cuda', 0))


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().contiguous().view(torch.int32).cpu().numpy()


def _flags_clear(eng):
    torch.cuda.synchronize()
    eng.raise_if_error()
    assert eng.poll_saturation(warn=False) == 0


@contextlib.contextmanager
def _poisoned_empty(byte: int):
    """Every float32 / uint8 tensor torch.empty returns inside the block starts as ``byte`` in every byte."""
    real = torch.empty

    def empty(*args, **kw):
        t = real(*args, **kw)
        if t.is_cuda and t.dtype in (torch.float32, torch.uint8):
            t.view(torch.uint8).fill_(byte)
        return t

    torch.empty = empty
    try:
        yield
    finally:
        torch.empty = real


@pytest.mark.parametrize('engine', ENGINES)
def test_block1_output_does_not_depend_on_batch_or_position(model, pool, engine):
    eng = _engine(model, engine)
    alone = np.stack([_bits(eng.debug_forward_until(pool[i:i + 1], BLOCK1))[0] for i in range(POOL)])
    rng = np.random.default_rng(engine)
    for b in BATCHES:
        idx = rng.integers(0, POOL, b)
        got = _bits(eng.debug_forward_until(pool[torch.from_numpy(idx).cuda()], BLOCK1))
        bad = [int(i) for i in np.flatnonzero((got != alone[idx]).reshape(b, -1).any(axis=1))]
        assert not bad, f'batch {b}: faces {bad[:8]} differ from the same crops run alone'
    _flags_clear(eng)


def _framed(u8: torch.Tensor, m: int) -> torch.Tensor:
    """CenterCrop(m) of the reference loader: a frame of m pixels set to 0."""
    out = u8.clone()
    if m > 0:
        out[..., :m, :] = 0
        out[..., -m:, :] = 0
        out[..., :, :m] = 0
        out[..., :, -m:] = 0
    return out


@pytest.mark.parametrize('margin', [0, 1, 7])
@pytest.mark.parametrize('engine', ENGINES)
def test_uint8_crops_match_fp32_crops(model, engine, margin):
    eng = _engine(model, engine)
    u8 = synthetic.make_structured_crops_u8(133, seed=40 + margin)
    eng.set_center_crop(margin)
    try:
        lmk_u8, p_u8 = eng.forward_landmarks(u8.cuda(), want_params=True)
    finally:
        eng.set_center_crop(0)
    lmk_f, p_f = eng.forward_landmarks(synthetic.normalize_crops(_framed(u8, margin)).cuda(), want_params=True)
    assert np.array_equal(_bits(p_u8), _bits(p_f))
    assert np.array_equal(_bits(lmk_u8), _bits(lmk_f))
    if margin > 0:     # the border changes the result: the frame really was applied
        lmk_plain, _ = eng.forward_landmarks(synthetic.normalize_crops(u8).cuda(), want_params=True)
        assert not np.array_equal(_bits(lmk_plain), _bits(lmk_f))
    _flags_clear(eng)


@pytest.mark.parametrize('engine', ENGINES)
def test_stale_and_poisoned_workspaces(model, pool, engine):
    eng = _engine(model, engine)
    x = pool[torch.arange(133, device='cuda') % POOL]
    u8 = synthetic.make_structured_crops_u8(133, seed=9)
    r0 = _bits(eng.debug_forward_until(x, BLOCK1))
    p0 = _bits(eng.forward_landmarks(u8.cuda(), want_params=True)[1])
    # a larger call leaves plausible stale bytes past the batch in every workspace
    eng.debug_forward_until(seeded_crops(300, 4), BLOCK1)
    eng.forward_landmarks(synthetic.make_structured_crops_u8(300, seed=5).cuda())
    assert np.array_equal(_bits(eng.debug_forward_until(x, BLOCK1)), r0)
    assert np.array_equal(_bits(eng.forward_landmarks(u8.cuda(), want_params=True)[1]), p0)
    _flags_clear(eng)
    for byte in (0xFF, 0x7F):
        assert eng.debug_fill_workspaces(byte) > 0
        with _poisoned_empty(byte):
            got = _bits(eng.debug_forward_until(x, BLOCK1))
        assert np.array_equal(got, r0), f'fill {byte:#x}: block-1 output differs'
        eng.debug_fill_workspaces(byte)
        with _poisoned_empty(byte):
            got = _bits(eng.forward_landmarks(u8.cuda(), want_params=True)[1])
        assert np.array_equal(got, p0), f'fill {byte:#x}: uint8 params differ'
        _flags_clear(eng)
