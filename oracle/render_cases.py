"""TEST INFRASTRUCTURE ONLY -- meshes at the edges of the Sim3DR rasteriser's arithmetic, shared by the CPU emulation
tests and the GPU oracle tests, and the host-side pixel boxes of the frame-axis plan with the reference's conversions.

The reference (``Sim3DR/lib/rasterize_kernel.cpp``) is baseline x86-64 code: ``(int)`` of a float at or beyond 2^31, or of
NaN, is ``cvttss2si``'s INT_MIN, so a triangle whose largest x or y is that far away gets an empty box and is skipped,
and a colour whose ``255 * colour`` is that large is written as byte 0.  ``out_of_range_cases`` puts every such value
(and the ones just inside the range) on a vertex coordinate, a depth and a colour, next to degenerate triangles.
"""
from __future__ import annotations

import numpy as np

INT_MIN = -2 ** 31
F_BELOW_2_31 = float(np.nextafter(np.float32(2 ** 31), np.float32(0)))      # 2^31 - 128: the largest float that converts
CANVAS = (24, 32)                                                              # h, w of the cases below


def x86_int(a) -> np.ndarray:
    """``(int)`` of float32 values as x86-64 computes it: truncation in [-2^31, 2^31), INT_MIN elsewhere (NaN too)."""
    a = np.asarray(a, np.float32)
    ok = (a >= np.float32(-2 ** 31)) & (a < np.float32(2 ** 31))
    return np.where(ok, np.trunc(np.where(ok, a, 0)).astype(np.int64), INT_MIN)


def tri_boxes(ver: np.ndarray, tri: np.ndarray, h: int, w: int):
    """Per triangle the clamped box ``(x0, y0, x1, y1)`` of the reference's loop (:245-249) and whether it is drawn."""
    x, y = ver[:, 0][tri], ver[:, 1][tri]

    def fmin(c):                                      # std::min(a, std::min(b, c)): the comparison form, NaN-order dependent
        m = np.where(c[:, 2] < c[:, 1], c[:, 2], c[:, 1])
        return np.where(m < c[:, 0], m, c[:, 0])

    def fmax(c):
        m = np.where(c[:, 1] < c[:, 2], c[:, 2], c[:, 1])
        return np.where(c[:, 0] < m, m, c[:, 0])

    with np.errstate(invalid='ignore'):
        x0 = np.maximum(x86_int(np.floor(fmin(x))), 0)
        x1 = np.minimum(x86_int(np.ceil(fmax(x))), w - 1)
        y0 = np.maximum(x86_int(np.floor(fmin(y))), 0)
        y1 = np.minimum(x86_int(np.ceil(fmax(y))), h - 1)
    return np.stack([x0, y0, x1, y1], 1), (x1 >= x0) & (y1 >= y0)


def mesh_box(ver: np.ndarray, tri: np.ndarray, h: int, w: int):
    """Union of the drawn triangles' boxes of one (nver,3) mesh, ``[0, 0, -1, -1]`` if none is drawn, and its area."""
    b, live = tri_boxes(ver, tri, h, w)
    if not live.any():
        return [0, 0, -1, -1], 0
    b = b[live]
    box = [int(b[:, 0].min()), int(b[:, 1].min()), int(b[:, 2].max()), int(b[:, 3].max())]
    return box, (box[2] - box[0] + 1) * (box[3] - box[1] + 1)


def _case(ver, tri, col=None):
    ver = np.asarray(ver, np.float32)
    if col is None:
        col = np.tile(np.array([[0.9, 0.5, 0.2]], np.float32), (ver.shape[0], 1))
        col[1::2] = (0.1, 0.7, 0.4)
    return ver, np.asarray(tri, np.int32), np.asarray(col, np.float32)


def out_of_range_cases():
    """``[(name, vertices (n,3) f32, triangles (k,3) i32, colours (n,3) f32)]`` on a ``CANVAS`` canvas.  Every case also
    draws an ordinary triangle that overlaps the special one, so the image shows whether the special one was drawn."""
    inf, nan = float('inf'), float('nan')
    near = [F_BELOW_2_31, 2.0 ** 31, 3e9, 1e18, inf]
    base = [[0, 0, 1], [20, 0, 1], [0, 20, 1], [4, 2, -5], [30, 6, -5], [8, 22, -5]]
    other = [3, 4, 5]
    cases = []
    for axis, corner, name in ((0, 1, 'x'), (1, 2, 'y')):
        for v in [s * a for a in near for s in (1, -1)] + [nan]:
            ver = np.array(base, np.float64)
            ver[corner, axis] = v
            tag = {F_BELOW_2_31: '2^31-128', 2.0 ** 31: '2^31'}.get(abs(v), f'{abs(v):g}')
            cases.append(_case(ver, [[0, 1, 2], other]) + (f'vertex_{name}={"-" if v < 0 else ""}{tag}',))
            if v == 3e9 or v != v:                                     # the same value on the first corner: min and max order
                ver2 = ver[[corner, 0, 3 - corner, 3, 4, 5]]
                cases.append(_case(ver2, [[0, 1, 2], other]) + (f'vertex_{name}={tag}_first',))
    for z, tag in ((-1e8, '-1e8'), (float(np.nextafter(np.float32(-1e8), np.float32(0))), 'above_-1e8'), (inf, 'inf'),
                   (-inf, '-inf'), (nan, 'nan'), (0.0, '+0'), (-0.0, '-0')):
        ver = np.array(base, np.float64)
        ver[:3, 2] = z
        cases.append(_case(ver, [[0, 1, 2], other]) + (f'depth={tag}',))
        ver = np.array(base, np.float64)
        ver[0, 2] = z                                                  # one corner only: interpolated across the face
        cases.append(_case(ver, [[0, 1, 2], other]) + (f'depth_corner={tag}',))
    for c, tag in ((-1e10, '-1e10'), (-0.5, '-0.5'), (1.5, '1.5'), (8421504.0, '8421504'), (8421505.0, '8421505'), (1e10, '1e10'),
                   (inf, 'inf'), (-inf, '-inf'), (nan, 'nan')):
        ver = np.array(base, np.float64)
        col = np.full((6, 3), 0.25, np.float32)
        col[:3, 0] = c                                                 # constant over the face
        col[0, 1] = c                                                  # one corner: a ramp from c down to 0.5
        col[1:3, 1] = 0.5
        cases.append(_case(ver, [[0, 1, 2], other], col) + (f'colour={tag}',))
    degenerate = {
        'repeated_index': ([[2, 3, 2], [12, 15, 3], [0, 0, 0]], [[0, 0, 1], [0, 1, 2]]),
        'repeated_position': ([[2, 3, 2], [2, 3, 4], [12, 15, 3]], [[0, 1, 2], [1, 2, 0]]),
        'collinear': ([[1, 1, 2], [11, 11, 3], [21, 21, 4], [5, 1, 0], [25, 9, 0], [3, 18, 0]], [[0, 1, 2], [3, 4, 5]]),
        'den_underflow': ([[0, 0, 1], [1e-20, 0, 1], [0, 1e-20, 1], [2, 3, 0]], [[0, 1, 2], [3, 1, 2]]),
    }
    for name, (ver, tri) in degenerate.items():
        cases.append(_case(ver, tri) + (name,))
    return [(name, ver, tri, col) for ver, tri, col, name in cases]
