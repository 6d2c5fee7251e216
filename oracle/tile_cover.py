"""Batch sizes and face subsets that put every tile kind of the fused backbone kernels under a check.  TEST
INFRASTRUCTURE.

The fused MobileNetV2 blocks tile a batch into face groups of 1, 2 or 4 faces (``fused_tile_plan`` in
``kernels_fused.cuh``, read here through ``syn_debug_tile_plan``) and run them on a persistent grid of
min(tiles, SMs) CTAs; the tail kernel takes 8-face tiles over ``ctas_per_slice`` CTAs per channel slice
(``synergy_b200.cu``).  Which tiles exist depends on the batch and on the SM count (132 on an H100 SXM, 114 on a PCIe
card), so the batches are derived from the SM count and every one is checked to produce the plan it is meant for:

  mixed_pairs   full waves of two-face groups, then a tail wave of single-face groups (split = a multiple of the SM
                count, at least two single-face groups);
  odd_pairs     every group two-face plus one odd face (split = B // 2); its last 8-face tail tile is ragged and there
                are more tail tiles than ``ctas_per_slice``;
  ragged_quads  more four-face groups than SMs, the last one holding 3 faces.

With any of them the one-face blocks also run several tiles per CTA.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Tuple

import torch

TAIL_FACES = 8          # kTailFaces (csrc/kernels_tail.cuh)


def tile_plan(batch: int, sms: int, faces_per_tile: int) -> Tuple[int, int]:
    """(split, face_groups) of the fused kernels for a batch on ``sms`` SMs."""
    from synergynet_b200 import _lib
    split, groups = C.c_int(-1), C.c_int(-1)
    _lib.check(_lib.load().syn_debug_tile_plan(batch, sms, faces_per_tile, C.byref(split), C.byref(groups)))
    return split.value, groups.value


def tail_ctas_per_slice(batch: int, sms: int) -> int:
    """CTAs per channel slice of ``tail_conv_pool_kernel`` (run_backbone in synergy_b200.cu)."""
    ntiles = -(-batch // TAIL_FACES)
    return max(1, min(ntiles, sms // 10))


def choose_batches(sms: int) -> Dict[str, int]:
    odd = 3 * sms // 2 | 1
    while odd % TAIL_FACES == 0 or -(-odd // TAIL_FACES) <= tail_ctas_per_slice(odd, sms):
        odd += 2
    return {'mixed_pairs': 2 * sms + 2 * (sms // 4), 'odd_pairs': odd, 'ragged_quads': 4 * sms + 3}


def check_plan(kind: str, batch: int, sms: int) -> None:
    """Assert that ``batch`` produces the tile plan ``kind`` names."""
    split, groups = tile_plan(batch, sms, 2)
    if kind == 'mixed_pairs':
        assert split >= sms and split % sms == 0 and split < batch // 2, (batch, sms, split)
        assert groups - split >= 2 and groups > sms, (batch, sms, split, groups)
    elif kind == 'odd_pairs':
        assert batch % 2 == 1 and split == batch // 2 and groups == split + 1, (batch, sms, split, groups)
        tail_tiles = -(-batch // TAIL_FACES)
        assert batch % TAIL_FACES != 0 and tail_tiles > tail_ctas_per_slice(batch, sms), (batch, sms)
    elif kind == 'ragged_quads':
        _, g4 = tile_plan(batch, sms, 4)
        assert g4 > sms and batch - 4 * (g4 - 1) == 3, (batch, sms, g4)
    else:
        raise ValueError(kind)


def faces_to_check(batch: int, sms: int, seed: int = 0, n_random: int = 4) -> List[int]:
    """A face subset that covers every tile kind of the batch: face 0; both faces of the last two-face group; the
    first and last single-face groups; every face of the last (possibly ragged) four-face group; faces whose tile is a
    CTA's second or later tile, for 1-, 2- and 4-face groups and for the tail kernel; a few seeded random faces."""
    faces = {0, batch - 1}
    split, groups = tile_plan(batch, sms, 2)
    if split > 0:
        faces |= {2 * split - 2, 2 * split - 1}
    if groups > split:
        faces |= {2 * split, batch - 1}
    if groups > sms:                                       # group index >= SMs: its tiles come after the first wave
        faces.add(2 * sms if sms < split else 2 * split + (sms - split))
    _, g4 = tile_plan(batch, sms, 4)
    faces |= set(range(4 * (g4 - 1), batch))
    if g4 > sms:
        faces.add(4 * sms)
    if batch > sms:
        faces.add(sms)                                     # one-face groups
    cps = tail_ctas_per_slice(batch, sms)
    if TAIL_FACES * cps < batch:
        faces.add(TAIL_FACES * cps)
    g = torch.Generator().manual_seed(seed)
    faces |= set(torch.randint(0, batch, (n_random,), generator=g).tolist())
    return sorted(faces)
