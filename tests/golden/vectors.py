"""The golden vectors of the reference (recorded by ``tests/golden/make_golden.py``), stored as several ``.npz`` files so
that each stays under 1 MB: ``ref_vectors.npz`` (everything below), ``ref_vectors_scene.npz`` (the ``get_all_outputs``
scene: ``scene*``) and ``ref_vectors_lmk1024.npz`` (landmarks of the 1024-face batch).  Tests read them as one dict."""
import os

import numpy as np

DIR = os.path.dirname(os.path.abspath(__file__))
MAIN = 'ref_vectors.npz'


def part_of(key: str) -> str:
    if key.startswith('scene'):
        return 'ref_vectors_scene.npz'
    if key == 'lmk1024':
        return 'ref_vectors_lmk1024.npz'
    return MAIN


PARTS = (MAIN, 'ref_vectors_scene.npz', 'ref_vectors_lmk1024.npz')


def load_ref_vectors() -> dict:
    out = {}
    for name in PARTS:
        out.update(dict(np.load(os.path.join(DIR, name), allow_pickle=False)))
    return out


def save_ref_vectors(arrays: dict, directory: str = DIR) -> None:
    for name in PARTS:
        np.savez_compressed(os.path.join(directory, name), **{k: v for k, v in arrays.items() if part_of(k) == name})
