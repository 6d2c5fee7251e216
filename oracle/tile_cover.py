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

``placement`` / ``check_placement`` lay a pool of distinct faces over a batch so that every pool face is computed in
several tile slots, and state which slots and tile kinds of a batch's plans the pool faces reach.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Tuple

import torch

TAIL_FACES = 8          # kTailFaces (csrc/kernels_tail.cuh)
ROW_TILE = 128          # rows of a tc_gemm_kernel CTA tile (csrc/kernels_tc.cuh), the unfused engines' GEMMs
MAP_PIXELS = (3600, 900, 225, 64, 16)       # pixels per face of the backbone's maps: 60x60, 30x30, 15x15, 8x8, 4x4


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


def placement(batch: int, pool: int) -> torch.Tensor:
    """The pool face of every face of a batch: face b is pool face (b + b // pool) % pool.  Each repetition of the pool
    is shifted by one more face, so from one repetition to the next a pool face moves to the next slot of the 2-, 4- and
    8-face tiles, and to another row offset of the 128-row GEMM tiles."""
    b = torch.arange(batch)
    return (b + b // pool) % pool


def check_placement(batch: int, sms: int, pool: int) -> Tuple[Dict[str, List[int]], Dict[str, str]]:
    """Where the pool faces of ``placement(batch, pool)`` land in the tile plans of ``batch`` on ``sms`` SMs.

    Returns (met, dropped).  ``met`` maps every claim the batch meets to the pool faces that witness it, ``dropped`` maps
    every other claim to the reason the batch cannot meet it:

      pair_both_slots     a pool face sits in slot 0 of one two-face group and in slot 1 of another;
      single_face_group   pool faces sit in single-face groups (the tail wave, or the odd face, of the two-face plan);
      quad_every_slot     a pool face sits in each of the four slots of four-face groups;
      quad_ragged_last    pool faces sit in the last four-face group, which holds fewer than four faces;
      tail_every_slot     a pool face sits in each of the 8 slots of the tail kernel's tiles;
      later_tile_one      faces in a CTA's second or later tile of the one-face blocks (one tile per face and strip);
      later_tile_pair     the same for the two-face blocks (one tile per face group);
      later_tile_quad     the same for the four-face blocks;
      later_tile_tail     the same for the tail kernel (tiles pi + i * ctas_per_slice);
      rows<px>            at the map size of px pixels per face, the faces start at every row offset (b * px) % 128 can
                          take; the witnesses are the pool faces that start at two or more offsets.
    """
    place = placement(batch, pool).tolist()
    met: Dict[str, List[int]] = {}
    dropped: Dict[str, str] = {}

    def claim(name: str, faces, reason: str) -> None:
        faces = sorted(set(faces))
        if faces:
            met[name] = faces
        else:
            dropped[name] = reason

    def every_slot(faces: range, slots: int) -> List[int]:
        seen: Dict[int, set] = {}
        for b in faces:
            seen.setdefault(place[b], set()).add(b % slots)
        return [p for p, s in seen.items() if len(s) == slots]

    split, groups = tile_plan(batch, sms, 2)
    _, g4 = tile_plan(batch, sms, 4)
    cps = tail_ctas_per_slice(batch, sms)
    claim('pair_both_slots', every_slot(range(2 * split), 2),
          'no two-face groups' if split == 0 else f'the {2 * split} faces of the two-face groups hold no pool face twice')
    claim('single_face_group', (place[b] for b in range(2 * split, batch)), f'every face is in a two-face group (B = {batch})')
    claim('quad_every_slot', every_slot(range(batch), 4), f'B = {batch} < 3 * P + 4: no pool face reaches all four slots')
    claim('quad_ragged_last', (place[b] for b in range(4 * (g4 - 1), batch)) if batch % 4 else (),
          f'B = {batch} is a multiple of 4: the last four-face group is full')
    claim('tail_every_slot', every_slot(range(batch), TAIL_FACES),
          f'B = {batch} < 7 * P + 8: no pool face reaches all 8 slots of a tail tile')
    claim('later_tile_one', (place[b] for b in range(sms, batch)), f'B = {batch} <= {sms} SMs')
    first_late = 2 * sms if sms <= split else 2 * split + (sms - split)      # first face of two-face-plan group `sms`
    claim('later_tile_pair', (place[b] for b in range(first_late, batch)) if groups > sms else (),
          f'{groups} face groups <= {sms} SMs: every CTA runs one tile')
    claim('later_tile_quad', (place[b] for b in range(4 * sms, batch)) if g4 > sms else (),
          f'{g4} four-face groups <= {sms} SMs: every CTA runs one tile')
    claim('later_tile_tail', (place[b] for b in range(TAIL_FACES * cps, batch)),
          f'{-(-batch // TAIL_FACES)} tail tiles <= {cps} CTAs per channel slice')
    for px in MAP_PIXELS:
        n_off = ROW_TILE // math.gcd(px, ROW_TILE)
        offsets: Dict[int, set] = {}
        for b in range(batch):
            offsets.setdefault(place[b], set()).add(b * px % ROW_TILE)
        reached = set().union(*offsets.values())
        claim(f'rows{px}', [p for p, o in offsets.items() if len(o) > 1] if len(reached) == n_off else (),
              f'the faces start at {len(reached)} of the {n_off} row offsets of a {px}-pixel map'
              if len(reached) < n_off else f'no pool face starts at two row offsets of a {px}-pixel map')
    return met, dropped
