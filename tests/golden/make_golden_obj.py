"""Writes tests/golden/obj_golden.npz and obj_golden.json: the files the reference's own ``write_obj``
(utils/inference.py:8-23) and ``write_obj_with_colors`` (artistic.py:19-31, the same function as
uv_texture_realFaces.py:21-33) write for seeded meshes.  Run where the reference tree is present:

    python tests/golden/make_golden_obj.py

The two functions are taken from the reference sources at generation time: their definitions are read with ``ast`` and
executed alone, so the modules' other imports (matplotlib, torch, cv2, the model) are never loaded; nothing from this
repository computes a recorded value.  The npz holds the inputs, the json the name of the file each call wrote and the
sha256 and size of its bytes.  The meshes carry the edge values of the '{:.4f}' field (4-decimal ties, signed zeros,
NaNs with both signs and several payloads, infinities, subnormals, 1e20, FLT_MAX); the triangles come as int32, int64
and integral float64, the colours as uint8 and as float32 from uint8.
"""
import ast
import hashlib
import json
import os
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('SYNERGYNET_REF', os.path.join(os.sep, 'root', 'reference'))
OUT_NPZ = os.path.join(HERE, 'obj_golden.npz')
OUT_JSON = os.path.join(HERE, 'obj_golden.json')


def edge_values() -> np.ndarray:
    """float32 values on the edges of '{:.4f}'."""
    bits = [0x00000000, 0x80000000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFBFFFFF, 0x7FA5A5A5, 0x7F800000, 0xFF800000,
            0x00000001, 0x80000001, 0x007FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF]
    v = np.array(bits, np.uint32).view(np.float32)
    ties = np.array([1, 3, 5, 7, 9, 11, 13, 15, 31, 33, 63, 65, 1023, 1025, 99999, (1 << 24) - 1], np.float64) / 32
    other = np.array([-1e-5, 1e-5, 0.00005, -0.00005, 0.00015, 1e20, -1e20, 2.0 ** 24, 2.0 ** 23 + 1, 0.5, 1.0, -1.0, 9.99995,
                      99999.99995, 123456.789, 2.0 ** -15, 2.0 ** -14 * 3], np.float64)
    return np.concatenate([v, ties.astype(np.float32), -ties.astype(np.float32), other.astype(np.float32)])


def make_cases(rng):
    """[(kind, arrays)]; kind 'obj' or 'colors'."""
    cases = []
    for k, (n, ntri, tri_dtype) in enumerate([(300, 500, np.int64), (257, 256, np.int32), (64, 90, np.float64), (1, 1, np.int64)]):
        v = np.stack([rng.uniform(-50, 700, n), rng.uniform(-50, 500, n), rng.normal(0, 60, n)]).astype(np.float32)
        if k == 0:
            e = edge_values()
            v[:, :e.size] = np.stack([e, np.roll(e, 1), np.roll(e, 2)])
        tri = rng.integers(0, 60000, (3, ntri))
        tri[:, 0] = (0, 1, 53214)
        cases.append(('obj', {'vertices': v, 'triangles': tri.astype(tri_dtype)}))
    for k, (n, keep_n, ntri, tri_dtype, col_f32) in enumerate([(400, 333, 300, np.int64, False), (400, 333, 300, np.float64, True),
                                                                (200, 200, 150, np.int32, True)]):
        v = np.stack([rng.uniform(0, 640, n), rng.uniform(0, 480, n), rng.normal(0, 50, n)]).astype(np.float32)
        if k == 0:
            e = edge_values()
            v[:, :e.size] = np.stack([np.roll(e, 3), e, np.roll(e, 5)])
        keep = np.sort(rng.choice(n, keep_n, replace=False)).astype(np.int64)
        col = rng.integers(0, 256, (n, 3)).astype(np.uint8)
        col[0] = (0, 255, 7)
        tri = rng.integers(1, keep_n + 1, (3, ntri)).astype(tri_dtype)
        cases.append(('colors', {'vertices': v, 'keep': keep, 'triangles': tri, 'colors_u8': col, 'colors_f32': np.array([int(col_f32)])}))
    return cases


def reference_functions():
    """write_obj and write_obj_with_colors from the reference sources, their definitions executed alone."""
    def grab(rel, name):
        src = open(os.path.join(REF, rel)).read()
        node = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == name)
        return ast.get_source_segment(src, node)
    a, b = grab('artistic.py', 'write_obj_with_colors'), grab('uv_texture_realFaces.py', 'write_obj_with_colors')
    assert a == b, 'the two write_obj_with_colors differ'
    scope = {}
    exec(grab('utils/inference.py', 'write_obj') + '\n' + a, scope)
    return scope['write_obj'], scope['write_obj_with_colors']


def main():
    write_obj, write_obj_with_colors = reference_functions()
    rng = np.random.default_rng(20261018)
    arrays, doc = {}, {'numpy': np.__version__, 'cases': []}
    tmp = tempfile.mkdtemp(prefix='obj_golden_')
    names = ['mesh', 'mesh.obj', 'a.b', 'face.v2.obj', 'x.OBJ', 'y.', 'z.obj.obj']
    for i, (kind, a) in enumerate(make_cases(rng)):
        for k, v in a.items():
            arrays[f'{k}{i}'] = v
        name = names[i % len(names)]
        before = set(os.listdir(tmp))
        if kind == 'obj':
            write_obj(os.path.join(tmp, name), a['vertices'], a['triangles'])
        else:
            col = a['colors_u8'][a['keep']]
            col = col.astype(np.float32) if a['colors_f32'][0] else col
            write_obj_with_colors(os.path.join(tmp, name), a['vertices'][:, a['keep']], a['triangles'], col)
        (written,) = set(os.listdir(tmp)) - before
        data = open(os.path.join(tmp, written), 'rb').read()
        os.remove(os.path.join(tmp, written))
        doc['cases'].append({'kind': kind, 'name': name, 'written': written, 'bytes': len(data),
                             'sha256': hashlib.sha256(data).hexdigest()})
    np.savez_compressed(OUT_NPZ, **arrays)
    with open(OUT_JSON, 'w') as f:
        json.dump(doc, f, indent=1)
        f.write('\n')
    print('wrote', OUT_NPZ, OUT_JSON, len(doc['cases']), 'cases')


if __name__ == '__main__':
    main()
