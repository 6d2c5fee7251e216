"""Writes tests/golden/draw_digests.json: the sha256 of the images cv2.line(img, p0, p1, colour, 4) leaves after drawing
seeded sequences of segments onto seeded canvases (draw_cases below), so a host without OpenCV still holds the line
emulation (csrc/draw_math.h) to OpenCV's bytes.  Run with OpenCV 4.x:

    python tests/golden/make_golden_draw.py
"""
import hashlib
import json
import os

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'draw_digests.json')
SIZES = ((1, 1), (1, 23), (17, 1), (37, 53), (64, 64), (9, 200), (31, 30))


def _point(rng, h, w):
    kind = rng.integers(0, 6)
    if kind == 0:                                              # inside
        return [int(rng.integers(0, w)), int(rng.integers(0, h))]
    if kind == 1:                                              # on, just inside or just outside a border
        near = lambda n: int(rng.choice([-5, -4, -3, -2, -1, 0, 1, 2, n - 3, n - 2, n - 1, n, n + 1, n + 2, n + 3, n + 4]))
        return [near(w), near(h)]
    if kind == 2:                                              # around the canvas
        return [int(rng.integers(-3 * w - 8, 4 * w + 8)), int(rng.integers(-3 * h - 8, 4 * h + 8))]
    if kind == 3:                                              # far outside: 64-bit fixed point
        return [int(rng.integers(-(1 << 30), (1 << 30) + 1)), int(rng.integers(-(1 << 30), (1 << 30) + 1))]
    if kind == 4:                                              # the int32 edges
        return [int(rng.choice([-(1 << 31), (1 << 31) - 1, -(1 << 30), 1 << 30])), int(rng.integers(-4, h + 4))]
    return [int(rng.integers(-2, w + 2)), int(rng.choice([-(1 << 31), (1 << 31) - 1, -(1 << 30), 1 << 30]))]


def _segment(rng, h, w):
    p0 = _point(rng, h, w)
    kind = rng.integers(0, 5)
    if kind == 0:                                              # length 0
        p1 = list(p0)
    elif kind == 1:                                            # length 1, any of the 8 neighbours
        d = [(1, 0), (1, 1), (0, 1), (-1, 1), (-1, 0), (-1, -1), (0, -1), (1, -1)][rng.integers(0, 8)]
        p1 = [min(max(p0[0] + d[0], -(1 << 31)), (1 << 31) - 1), min(max(p0[1] + d[1], -(1 << 31)), (1 << 31) - 1)]
    elif kind == 2:                                            # a short one in a random octant
        a, r = rng.uniform(0, 2 * np.pi), rng.uniform(1, 12)
        p1 = [int(np.clip(p0[0] + round(r * np.cos(a)), -(1 << 31), (1 << 31) - 1)),
              int(np.clip(p0[1] + round(r * np.sin(a)), -(1 << 31), (1 << 31) - 1))]
    else:
        p1 = _point(rng, h, w)
    colour = [int(c) for c in rng.integers(0, 256, 3)]
    return p0 + p1 + [colour[0] | (colour[1] << 8) | (colour[2] << 16)]


def draw_cases(seed, n_canvases, max_segments, sizes=SIZES):
    """[(image, segments (n,5) int32 x0, y0, x1, y1, b | g << 8 | r << 16), ...]: seeded canvases with sequences of
    overlapping segments of different colours."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_canvases):
        h, w = sizes[i % len(sizes)]
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        segs = np.array([_segment(rng, h, w) for _ in range(int(rng.integers(1, max_segments + 1)))], np.int64).astype(np.int32)
        out.append((img, segs))
    return out


def cv2_draw(img, segs):
    import cv2
    img = img.copy()
    for x0, y0, x1, y1, c in segs.tolist():
        cv2.line(img, (x0, y0), (x1, y1), (c & 255, (c >> 8) & 255, (c >> 16) & 255), 4)
    return img


def digest(x):
    return hashlib.sha256(np.ascontiguousarray(x, np.uint8).tobytes()).hexdigest()


# the committed set: 600 small canvases and two 720 x 1080 frames
DIGEST_SETS = ((1, 600, 24, SIZES), (2, 2, 300, ((720, 1080),)))


def main():
    import cv2
    doc = {'opencv': cv2.__version__, 'sets': [list(s[:3]) + [[list(x) for x in s[3]]] for s in DIGEST_SETS], 'digests': []}
    for seed, n, m, sizes in DIGEST_SETS:
        doc['digests'].append([digest(cv2_draw(img, segs)) for img, segs in draw_cases(seed, n, m, sizes)])
    with open(OUT, 'w') as f:
        json.dump(doc, f, indent=0)
        f.write('\n')
    print('wrote', OUT)


if __name__ == '__main__':
    main()
