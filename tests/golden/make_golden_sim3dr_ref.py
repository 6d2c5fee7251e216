"""Record the reference's own Sim3DR C++ (``Sim3DR/lib/rasterize_kernel.cpp``, compiled by ``oracle/Makefile`` into
``oracle/_ref/libsim3dr_ref.so``) on the inputs of ``tests/test_oracle_render.py::test_port_equals_compiled_reference``
and store its outputs in ``tests/golden/sim3dr_ref_vectors.npz``.

Needs the reference tree (``make -C oracle ref``); the test itself only reads the stored vectors.  Image pixels are
stored where the depth buffer was written (rows mirrored when ``reverse``: the image is drawn upside down, the depth
buffer is not): every other pixel is the test's seeded background, untouched.

    python tests/golden/make_golden_sim3dr_ref.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import render_port as rp  # noqa: E402
from synergynet_b200 import synthetic  # noqa: E402

DEPTH_INIT = np.float32(-1e8)          # rasterize_kernel.cpp: the depth buffer starts at -1e8 (Sim3DR.rasterize)


def drawn_pixels(depth, reverse):
    """Image pixels the rasteriser wrote: depth-buffer cells that left their initial value, in image rows."""
    d = depth != DEPTH_INIT
    return d[::-1] if reverse else d


def inputs():
    """The mesh pair, a few huge / degenerate triangles, and per mesh the colours and background (seeded)."""
    tri = synthetic.make_render_topology(60, 70)
    verts = synthetic.make_render_meshes(2, 200, 240, seed=5, rows=60, cols=70, size=120)
    extra = np.array([[0, 4199, 2100], [10, 10, 500], [69, 4130, 35]], np.int32)
    tri = np.ascontiguousarray(np.concatenate([tri, extra]))
    rng = np.random.default_rng(3)
    per_mesh = []
    for b in range(2):
        ver = np.ascontiguousarray(verts[b].T)
        col = rng.uniform(0, 1, ver.shape).astype(np.float32)
        bg = rng.integers(0, 256, (200, 240, 3), dtype=np.uint8)
        per_mesh.append((ver, col, bg))
    return tri, per_mesh


def main():
    if not rp.have_ref():
        sys.exit('oracle/_ref/libsim3dr_ref.so is missing: run `make -C oracle ref` where the reference tree exists')
    tri, per_mesh = inputs()
    out = {}
    for b, (ver, col, bg) in enumerate(per_mesh):
        out[f'normals_{b}'] = rp.get_normal(ver, tri, 'ref')
        for rev in (0, 1):
            img, depth = rp.rasterize(ver, tri, col, bg.copy(), reverse=bool(rev), kind='ref', return_depth=True)
            out[f'depth_{b}_{rev}'] = depth
            out[f'pixels_{b}_{rev}'] = img[drawn_pixels(depth, rev)]
    fp = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'sim3dr_ref_vectors.npz')
    np.savez_compressed(fp, **out)
    print(fp, os.path.getsize(fp), 'bytes')


if __name__ == '__main__':
    main()
