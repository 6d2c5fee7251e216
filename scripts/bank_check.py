#!/usr/bin/env python
"""Design aid: shared-memory bank-conflict degree of the lane -> address mappings used by the fused MBConv
kernel (synergynet_b200/csrc/kernels_fused.cuh).  The formulas below restate the kernel's indexing.

Model: 32 banks x 4 B.  A 128-bit access is served per quarter-warp (8 lanes), a 64-bit access per half-warp
(16 lanes), a 32-bit access per warp; lanes reading the SAME address are merged (broadcast).  Degree 1 =
conflict-free, degree n = n wavefronts where 1 would do.

    python scripts/bank_check.py            # table for every fused configuration
"""
from itertools import product

CONFIGS = {   # name: (NC, W, STRIDE, RO)  -- hidden-channel chunk, input width, depthwise stride, output rows per tile
    'stem_block1': (32, 60, 1, 6), 'block2': (32, 60, 2, 6), 'block3': (16, 30, 1, 15), 'block4': (16, 30, 2, 15),
    'block5/6': (64, 15, 1, 15), 'block7': (64, 15, 2, 8), 'block8-11': (64, 8, 1, 8), 'block12/13': (64, 8, 1, 8),
    'block14': (64, 8, 2, 4), 'block15/16': (32, 4, 1, 4), 'block17': (32, 4, 1, 4),
}


def degree(addrs, width):
    """addrs: byte address per lane of ONE warp instruction (None = lane inactive); width: bytes per lane."""
    lanes_per_phase = {16: 8, 8: 16, 4: 32}[width]
    worst = 1
    for p0 in range(0, 32, lanes_per_phase):
        per_bank = {}
        for a in addrs[p0:p0 + lanes_per_phase]:
            if a is None:
                continue
            for b in range(a // 4, (a + width) // 4):
                per_bank.setdefault(b % 32, set()).add(b)      # distinct 4-byte words per bank
        if per_bank:
            worst = max(worst, max(len(v) for v in per_bank.values()))
    return worst


def window_pixel_stride(nc):
    return (nc + 4) * 4                                       # HS_STRIDE floats: NC + 4


def dw_octet_loads(nc, w, stride, swap):
    """Default depthwise item: 8 lanes along x (GX = 8) or 4 x 2 (GX = 4), one octet = two LDS.128 per pixel."""
    sp, hs_cols = window_pixel_stride(nc), w + 2
    wo = (w - 1) // stride + 1
    gx = 8 if wo >= 8 else 4
    worst = 1
    for first_quad in (0, 1):
        addrs = []
        for lane in range(32):
            l8 = lane & 7
            lx, ly = l8 % gx, l8 // gx
            q = first_quad ^ (1 if (swap and (l8 & 4)) else 0)
            pix = (2 * ly * stride) * hs_cols + lx * stride    # row pairs: ly-th pair of the quarter-warp
            addrs.append(pix * sp + q * 16 + (lane >> 3) * 32)  # lanes 8.. : another octet (32 B further)
        worst = max(worst, degree(addrs, 16))
    return worst


def dw_quad_loads(nc, w, mirrored):
    """Register-blocked item (stride 1): a unit = 8 lanes x 2 quads; lanes 4-7 mirrored (walk columns right to left)."""
    sp, hs_cols = window_pixel_stride(nc), w + 2
    xl = 8 if w >= 15 else 4
    worst = 1
    for ic in range(4):
        addrs = []
        for lane in range(32):
            l8, qh = lane & 7, (lane >> 3) & 1
            lx, ly = l8 % xl, l8 // xl
            mir = mirrored and (l8 & 4)
            col = 2 * lx + (3 - ic if mir else ic)
            row = 2 * ly
            addrs.append((row * hs_cols + col) * sp + qh * 16 + (lane >> 4) * 64)
        worst = max(worst, degree(addrs, 16))
    return worst


def a2_quad_stores(w, mirrored):
    """8-byte operand stores of the register-blocked item: A2 row m at (m/8)*128 + (m%8)*16 (+ quad half * 8)."""
    xl = 8 if w >= 15 else 4
    worst = 1
    for a in range(2):
        addrs = []
        for lane in range(16):                                  # one half-warp = one unit
            l8, qh = lane & 7, lane >> 3
            lx, ly = l8 % xl, l8 // xl
            mir = mirrored and (l8 & 4)
            m = (2 * ly) * w + 2 * lx + ((1 - a) if mir else a)
            addrs.append((m // 8) * 128 + (m % 8) * 16 + qh * 8)
        worst = max(worst, degree(addrs + [None] * 16, 8))
    return worst


def epi1_stores(nc):
    """EPI1: lane = pixel (consecutive window pixels), one STS.128 per channel quad."""
    sp = window_pixel_stride(nc)
    return degree([lane * sp for lane in range(32)], 16)


def main():
    print(f'{"block":12s} {"NC":>3s} {"W":>3s} {"S":>2s} | EPI1 st | DW octet ld (plain / quad-swap) | DW quad ld (plain / mirrored) | A2 8-byte st (plain / mirrored)')
    for name, (nc, w, s, ro) in CONFIGS.items():
        e = epi1_stores(nc)
        o0, o1 = dw_octet_loads(nc, w, s, False), dw_octet_loads(nc, w, s, True)
        if s == 1 and w in (8, 15, 30, 60):
            q0, q1 = dw_quad_loads(nc, w, False), dw_quad_loads(nc, w, True)
            a0, a1 = a2_quad_stores((w - 1) // s + 1, False), a2_quad_stores((w - 1) // s + 1, True)
            quad = f'{q0} / {q1}'.ljust(29) + f' | {a0} / {a1}'
        else:
            quad = '-'.ljust(29) + ' | -'
        print(f'{name:12s} {nc:3d} {w:3d} {s:2d} | {e:7d} | {f"{o0} / {o1}":31s} | {quad}')


if __name__ == '__main__':
    main()
