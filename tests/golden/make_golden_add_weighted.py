"""Writes tests/golden/add_weighted_digests.json: the bytes cv2.addWeighted(a, 1 - alpha, b, alpha, 0) gives for all
65 536 uint8 pairs (a, b), a = i // 256, b = i % 256, in the SIMD body of one long row and in the scalar path (rows of
three elements of a non-continuous array), as sha256 digests per alpha.  Run with OpenCV 4.x:

    python tests/golden/make_golden_add_weighted.py
"""
import hashlib
import json
import os

import numpy as np

ALPHAS = (0.0, 0.1, 0.3, 0.5, 0.6, 0.75, 1.0)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'add_weighted_digests.json')


def pairs():
    i = np.arange(65536)
    return (i // 256).astype(np.uint8), (i % 256).astype(np.uint8)


def cv2_body(a, b, alpha):
    """One continuous row: every element but OpenCV's last partial vector goes through the SIMD body."""
    import cv2
    return cv2.addWeighted(a.reshape(1, -1), 1 - alpha, b.reshape(1, -1), alpha, 0).reshape(-1)


def cv2_tail(a, b, alpha):
    """Rows of 3 elements with a 4-byte row step (not continuous): every element goes through the scalar loop."""
    import cv2
    pa, pb = np.zeros((a.size // 2, 4), np.uint8), np.zeros((b.size // 2, 4), np.uint8)
    pa[:, :2], pb[:, :2] = a.reshape(-1, 2), b.reshape(-1, 2)
    pa[:, 2], pb[:, 2] = a.reshape(-1, 2)[:, 0], b.reshape(-1, 2)[:, 0]
    out = cv2.addWeighted(pa[:, :3], 1 - alpha, pb[:, :3], alpha, 0)
    assert np.array_equal(out[:, 2], out[:, 0])
    return np.ascontiguousarray(out[:, :2]).reshape(-1)


def digest(x):
    return hashlib.sha256(np.ascontiguousarray(x, np.uint8).tobytes()).hexdigest()


def main():
    import cv2
    a, b = pairs()
    doc = {'opencv': cv2.__version__, 'pairs': 'a = i // 256, b = i % 256, i = 0..65535', 'alphas': list(ALPHAS),
           'body': {repr(al): digest(cv2_body(a, b, al)) for al in ALPHAS},
           'tail': {repr(al): digest(cv2_tail(a, b, al)) for al in ALPHAS}}
    with open(OUT, 'w') as f:
        json.dump(doc, f, indent=1)
        f.write('\n')
    print('wrote', OUT)


if __name__ == '__main__':
    main()
