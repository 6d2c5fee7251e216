"""Writes tests/golden/axis_golden.npz and axis_golden.json: what the reference's own ``draw_axis``
(utils/inference.py:199-244) draws, and raises, for seeded faces, called as singleImage.py:112-117 calls it -- once per
face, in order, on one image.  Run where the reference tree and OpenCV 4.x are present:

    python tests/golden/make_golden_axis.py

The reference module is imported from a scratch copy with matplotlib stubbed (tests/golden/make_golden.py does the same);
nothing from this repository computes a recorded value.  The npz holds the inputs (image sizes -- the images are base_image() -- angles as float64 -- Python
floats, as get_all_outputs returns them -- and float32 pts68), the json the sha256 of every resulting image, the name
of the exception raised (or null), and the number of cases on which a planner that keeps the end points in float64
(ignoring NumPy 2's scalar promotion) gives other integer points.
"""
import hashlib
import json
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
OUT_NPZ = os.path.join(HERE, 'axis_golden.npz')
OUT_JSON = os.path.join(HERE, 'axis_golden.json')


def face(rng, cx, cy, sx, sy):
    """(3,68) float32 landmarks: a jittered ellipse of half-extents sx, sy around (cx, cy)."""
    t = np.linspace(0, 2 * np.pi, 68, endpoint=False)
    p = np.stack([cx + sx * np.cos(t), cy + sy * np.sin(t), rng.normal(0, 10, 68)])
    p[:2] += rng.normal(0, 0.3, (2, 68)) * np.array([[sx], [sy]]) * 0.05
    return p.astype(np.float32)


def ends64(yaw, pitch, roll, pts68):
    """The end points with every term kept in float64 (the pre-NEP 50 result)."""
    pitch, yaw, roll = pitch * np.pi / 180, -(yaw * np.pi / 180), roll * np.pi / 180
    tdx, tdy = float(pts68[0, 30]), float(pts68[1, 30])
    size = math.sqrt((np.max(pts68[0]) - np.min(pts68[0])) * (np.max(pts68[1]) - np.min(pts68[1]))) * 0.5
    c, s = math.cos, math.sin
    return [size * (c(yaw) * c(roll)) + tdx, size * (c(pitch) * s(roll) + c(roll) * s(pitch) * s(yaw)) + tdy,
            size * (-c(yaw) * s(roll)) + tdx, size * (c(pitch) * c(roll) - s(pitch) * s(yaw) * s(roll)) + tdy,
            size * (s(yaw)) + tdx, size * (-c(yaw) * s(pitch)) + tdy]


def ends32(yaw, pitch, roll, pts68):
    """The same with the reference's types (float32 end points)."""
    pitch, yaw, roll = pitch * np.pi / 180, -(yaw * np.pi / 180), roll * np.pi / 180
    tdx, tdy = pts68[0, 30], pts68[1, 30]
    size = math.sqrt((np.max(pts68[0]) - np.min(pts68[0])) * (np.max(pts68[1]) - np.min(pts68[1]))) * 0.5
    c, s = math.cos, math.sin
    return [size * (c(yaw) * c(roll)) + tdx, size * (c(pitch) * s(roll) + c(roll) * s(pitch) * s(yaw)) + tdy,
            size * (-c(yaw) * s(roll)) + tdx, size * (c(pitch) * c(roll) - s(pitch) * s(yaw) * s(roll)) + tdy,
            size * (s(yaw)) + tdx, size * (-c(yaw) * s(pitch)) + tdy]


def int_or_none(v):
    try:
        return int(v)
    except (ValueError, OverflowError):
        return None


def differs64(yaw, pitch, roll, pts68):
    if not all(math.isfinite(a) for a in (yaw, pitch, roll)):
        return False
    with np.errstate(all='ignore'):
        return [int_or_none(v) for v in ends64(yaw, pitch, roll, pts68)] != [int_or_none(v) for v in ends32(yaw, pitch, roll, pts68)]


def make_cases(rng):
    """[(h, w, [(yaw, pitch, roll, pts68), ...]), ...]"""
    cases = []
    special = (0.0, 90.0, -90.0, 180.0, -180.0, 45.0, -30.0)
    for k, (yaw, pitch, roll) in enumerate([(a, b, c) for a in special[:5] for b in special[:5:2] for c in special[::3]]):
        cases.append((48, 64, [(yaw, pitch, roll, face(rng, 30 + k % 5, 22 + k % 3, 9 + k % 4, 11 - k % 3))]))
    for k in range(12):                                             # several faces, overlapping, some axes leaving
        n = 2 + k % 4
        faces = [(float(rng.uniform(-100, 100)), float(rng.uniform(-100, 100)), float(rng.uniform(-180, 180)),
                  face(rng, rng.uniform(-10, 75), rng.uniform(-10, 55), rng.uniform(3, 30), rng.uniform(3, 30))) for _ in range(n)]
        cases.append((50 + k, 70 - k, faces))
    wide = face(rng, 30, 20, 400, 300)                               # landmarks far wider than the image
    wide[:2, 30] = (30.0, 20.0)
    cases.append((40, 60, [(20.0, -10.0, 5.0, wide)]))
    flat = face(rng, 30, 20, 12, 9)
    flat[0] = flat[0, 30]                                            # all x equal: size 0, three zero-length lines
    line = face(rng, 25, 25, 12, 9)
    line[1] = 25.5                                                   # all y equal
    cases.append((40, 60, [(10.0, 20.0, 30.0, flat), (-10.0, 5.0, 60.0, line)]))
    one = face(rng, 0.4, 0.6, 0.2, 0.2)
    cases.append((1, 1, [(33.0, -12.0, 70.0, one)]))                 # a 1x1 canvas
    cases.append((1, 40, [(33.0, -12.0, 70.0, face(rng, 20, 0.5, 8, 0.4))]))
    cases.append((40, 1, [(-60.0, 12.0, -20.0, face(rng, 0.5, 20, 0.4, 8))]))
    # failures: a NaN angle, a NaN landmark, an infinite angle, and int32 overflow after one and after two axes
    cases.append((48, 64, [(10.0, 5.0, 0.0, face(rng, 30, 24, 10, 10)), (float('nan'), 5.0, 0.0, face(rng, 30, 24, 10, 10))]))
    bad = face(rng, 30, 24, 10, 10)
    bad[0, 30] = np.nan
    cases.append((48, 64, [(10.0, 5.0, 0.0, bad)]))
    cases.append((48, 64, [(float('inf'), 5.0, 0.0, face(rng, 30, 24, 10, 10))]))
    huge = face(rng, 30, 24, 3e9, 3e9)
    huge[:2, 30] = (30.0, 24.0)
    cases.append((48, 64, [(90.0, 0.0, 0.0, huge)]))                 # x axis drawn, then y overflows
    cases.append((48, 64, [(90.0, 0.0, 90.0, huge)]))
    # end points a float64 sum would round to another integer than the float32 one
    hits = 0
    while hits < 4:
        f = face(rng, rng.uniform(10, 50), rng.uniform(10, 40), rng.uniform(5, 25), rng.uniform(5, 25))
        ang = tuple(float(v) for v in rng.uniform(-90, 90, 3))
        if differs64(*ang, f):
            cases.append((48, 64, [(*ang, f)]))
            hits += 1
    return cases


def base_image(i, h, w):
    """The image case i draws on (regenerated by the tests rather than stored)."""
    y, x = np.mgrid[:h, :w]
    return np.stack([(x * 7 + y * 3 + i) % 256, (x * 2 + y * 11) % 256, np.full((h, w), 37 * i % 256)], -1).astype(np.uint8)


def main():
    import make_golden
    make_golden.scratch_reference()
    import cv2
    from utils.inference import draw_axis                     # the reference's own function
    rng = np.random.default_rng(20261017)
    cases = make_cases(rng)
    arrays, doc = {}, {'opencv': cv2.__version__, 'numpy': np.__version__, 'cases': []}
    n64 = 0
    for i, (h, w, faces) in enumerate(cases):
        img = base_image(i, h, w)
        arrays[f'hw{i}'] = np.array([h, w], np.int32)
        arrays[f'ang{i}'] = np.array([f[:3] for f in faces], np.float64)
        arrays[f'pts{i}'] = np.stack([f[3] for f in faces])
        canvas, err = img.copy(), None
        try:
            with np.errstate(all='ignore'):
                for yaw, pitch, roll, pts in faces:
                    res = draw_axis(canvas, yaw, pitch, roll, 0.0, 0.0, size=50, pts68=pts)
                    assert res is canvas
        except Exception as e:                                   # noqa: BLE001 -- the exception is what is recorded
            err = type(e).__name__
        n64 += any(differs64(*f) for f in faces)
        doc['cases'].append({'digest': hashlib.sha256(canvas.tobytes()).hexdigest(), 'error': err,
                             'changed': bool((canvas != img).any())})
    doc['float64_planner_differs'] = n64
    np.savez_compressed(OUT_NPZ, **arrays)
    with open(OUT_JSON, 'w') as f:
        json.dump(doc, f, indent=1)
        f.write('\n')
    print('wrote', OUT_NPZ, OUT_JSON, len(cases), 'cases;', n64, 'differ with a float64 planner;',
          sum(c['error'] is not None for c in doc['cases']), 'raise')


if __name__ == '__main__':
    main()
