"""The Sim3DR kernels on the H100 against the serial rasteriser, on seeded random meshes: the one-image canvas path
(``MeshRenderer.rasterize``: image and every mesh's depth buffer), the frame axis (``rasterize_frames`` and its plan),
normals and lighting.  The arbiter is the reference's own ``rasterize_kernel.cpp`` (``oracle/_ref``) where it was built,
and this project's C restatement of it always (they are also held to each other here).

The CPU emulation tests run the same ``render_math.h`` arithmetic through serial loops; what only the device can get
wrong is checked here: the thread-walked / warp-walked split of the triangle boxes at 64 pixels, the ballot loop over
warps of all-large, all-small and mixed triangles, the key atomics, the box-relative key addressing of the frame axis,
and the device's own float -> int conversions (``cvt.rzi`` saturates where x86 gives INT_MIN: render_math.h's
``to_int_x86``)."""
import functools

import numpy as np
import pytest
import torch

from oracle import render_cases as rc
from oracle import render_port as rp
from synergynet_b200 import Sim3DR, synthetic
from synergynet_b200.inference import RENDER_CFG

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
LIGHT_TOL = 2e-7                      # numpy's powf has no bit pattern to match (render_math.h, powi)


def serial(ver, tri, col, bg, reverse=False):
    """The meshes drawn one after the other onto ``bg`` by the serial rasteriser (the port, and the reference when built:
    both must agree).  Returns the image and every mesh's depth buffer (M,h,w)."""
    out, depths = [], []
    for kind in ['port'] + (['ref'] if rp.have_ref() else []):
        img, ds = bg.copy(), []
        with np.errstate(all='ignore'):
            for m in range(ver.shape[0]):
                img, d = rp.rasterize(ver[m], tri, col[m], img, reverse=reverse, kind=kind, return_depth=True)
                ds.append(d)
        out.append(img)
        depths.append(np.stack(ds) if ds else np.zeros((0,) + bg.shape[:2], np.float32))
    for img, d in zip(out[1:], depths[1:]):
        assert np.array_equal(img, out[0]) and np.array_equal(d, depths[0]), 'the port and the reference disagree'
    return out[0], depths[0]


def dev_vertices(ver, planar):
    """(M,nver,3) float32 on the device: interleaved, or a (M,3,nver) buffer read through a transposed view."""
    if planar:
        return torch.from_numpy(np.ascontiguousarray(ver.transpose(0, 2, 1))).to(DEV).transpose(1, 2)
    return torch.from_numpy(np.ascontiguousarray(ver)).to(DEV)


def plan_want(ver, tri, counts, h, w):
    boxes = [rc.mesh_box(ver[m], tri, h, w) for m in range(ver.shape[0])]
    return np.array([b for b, _ in boxes], np.int64).reshape(-1, 4), np.concatenate([[0], np.cumsum([a for _, a in boxes])])


# ---- (a), (b): random meshes -----------------------------------------------------------------------------------------------
CANVASES = [(1, 1), (1, 97), (97, 1), (255, 257), (40, 48), (17, 70)]
NTRI = [1, 31, 32, 33, 255, 256, 257]
NMESH = [1, 2, 5, 13, 40, 3, 8]
EDGE_BOXES = [(7, 9), (8, 8), (5, 13), (1, 63), (64, 1), (65, 1), (9, 7), (13, 5)]     # 63, 64 and 65 pixels
WARP_KINDS = ['small', 'large', 'mixed', 'edge']
N_CASES = 84


@functools.lru_cache(maxsize=None)
def scene(idx):
    """Case ``idx``: one topology and M meshes over it on an h x w canvas, with C-channel colours.  Triangles come in
    warps of 32 of one kind -- all small (boxes <= 36 px, walked by their own thread), all large, exactly 63 / 64 / 65
    pixel boxes, or a mix with whole-canvas, off-canvas and degenerate ones."""
    rng = np.random.default_rng(7000 + idx)
    h, w = CANVASES[idx % len(CANVASES)]
    ntri = NTRI[idx % len(NTRI)]
    nmesh = NMESH[idx % len(NMESH)] if h * w < 20000 else 1 + idx % 3
    c = (1, 3, 4)[idx % 3]
    planar, reverse, quant = bool(idx % 2), bool((idx // 2) % 2), bool((idx // 4) % 2)
    nver = 3 * ntri + 2
    tri = np.arange(3 * ntri, dtype=np.int32).reshape(ntri, 3)
    shared = rng.random(ntri) < 0.15                                   # some triangles share vertices / repeat corners
    tri[shared] = rng.integers(0, nver, (int(shared.sum()), 3))
    kinds = [WARP_KINDS[int(rng.integers(0, 4))] for _ in range((ntri + 31) // 32)]
    ver = np.empty((nmesh, nver, 3), np.float64)
    for m in range(nmesh):
        s = float(rng.choice([0.5, 1.0, 3.0]))
        ver[m, :, 0] = rng.uniform(-s * w * 0.3, w * (1 + 0.3 * s), nver)
        ver[m, :, 1] = rng.uniform(-s * h * 0.3, h * (1 + 0.3 * s), nver)
        ver[m, :, 2] = rng.uniform(-5, 5, nver)
        for i in np.flatnonzero(~shared):
            kind = kinds[i // 32]
            if kind == 'mixed':
                kind = ['small', 'large', 'edge', 'canvas', 'off', 'flat'][int(rng.integers(0, 6))]
            p = ver[m, 3 * i:3 * i + 3]
            if kind == 'small':
                p[:, :2] = rng.uniform([-2, -2], [w + 2, h + 2]) + rng.uniform(-2.5, 2.5, (3, 2))
            elif kind == 'edge':
                bw, bh = EDGE_BOXES[int(rng.integers(0, len(EDGE_BOXES)))]
                x, y = int(rng.integers(0, max(w - bw, 0) + 1)), int(rng.integers(0, max(h - bh, 0) + 1))
                a, b = int(rng.integers(0, bh)), int(rng.integers(0, bw))
                p[:, :2] = [[x, y + a], [x + bw - 1, y], [x + b, y + bh - 1]]
            elif kind == 'canvas':
                p[:, :2] = [[-w - 0.5, -h - 0.5], [3 * w + 0.5, -h], [-w, 3 * h + 0.5]]
            elif kind == 'off':
                p[:, 0] += 2 * w + 3
            elif kind == 'flat':
                p[1, :2] = p[0, :2]
        if quant:
            ver[m, :, :2] = np.round(ver[m, :, :2] * 2) / 2                # pixel centres on edges, and depth ties
            ver[m, :, 2] = np.round(ver[m, :, 2])
    ver = ver.astype(np.float32)
    if nmesh > 2:
        ver[1, :, 0] += 3 * w                                          # one mesh wholly off the canvas
    col = rng.uniform(0, 1, (nmesh, nver, c)).astype(np.float32)
    bg = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
    return dict(h=h, w=w, c=c, tri=tri, ver=ver, col=col, bg=bg, planar=planar, reverse=reverse, kinds=kinds)


def _id(idx):
    s = scene(idx)
    m, ntri = s['ver'].shape[0], s['tri'].shape[0]
    return (f'{idx}-{s["h"]}x{s["w"]}x{s["c"]}-m{m}-t{ntri}-{"planar" if s["planar"] else "inter"}'
            f'{"-rev" if s["reverse"] else ""}')


@pytest.mark.parametrize('idx', range(N_CASES), ids=_id)
def test_canvas_path_random_meshes(idx):
    s = scene(idx)
    r = Sim3DR.MeshRenderer(s['tri'], s['ver'].shape[1], DEV)
    img = torch.from_numpy(s['bg'].copy()).to(DEV)
    _, depth = r.rasterize(img, dev_vertices(s['ver'], s['planar']), torch.from_numpy(s['col']).to(DEV), reverse=s['reverse'],
                           return_depth=True)
    want, dwant = serial(s['ver'], s['tri'], s['col'], s['bg'], s['reverse'])
    got = img.cpu().numpy()
    assert np.array_equal(depth.cpu().numpy(), dwant), 'depth buffers'
    assert np.array_equal(got, want), f'image: {int((got != want).any(-1).sum())} pixels differ'


@pytest.mark.parametrize('idx', range(N_CASES), ids=_id)
def test_frame_axis_random_meshes(idx):
    """The same meshes spread over frames (some frames without a mesh): each frame's solid image is the serial drawing of
    its own meshes in order, and the plan's boxes and key offsets are the clipped boxes computed on the host."""
    s = scene(idx)
    ver, col, h, w, c = s['ver'], s['col'], s['h'], s['w'], s['c']
    rng = np.random.default_rng(idx)
    m = ver.shape[0]
    cuts = np.sort(rng.integers(0, m + 1, 3))                          # four frames, any of them may be empty
    counts = np.diff(np.concatenate([[0], cuts, [m]])).tolist()
    counts.insert(int(rng.integers(0, 5)), 0)                          # and one that is always empty
    frames = rng.integers(0, 256, (len(counts), h, w, c), dtype=np.uint8)
    r = Sim3DR.MeshRenderer(s['tri'], ver.shape[1], DEV)
    v = dev_vertices(ver, s['planar'])
    boxes, key_off = r.plan_frames(v, counts, h, w)
    want_boxes, want_off = plan_want(ver, s['tri'], counts, h, w)
    assert np.array_equal(boxes.cpu().numpy(), want_boxes) and key_off.cpu().numpy().tolist() == want_off.tolist()
    out = r.rasterize_frames(torch.from_numpy(frames).to(DEV), v, torch.from_numpy(col).to(DEV), counts).cpu().numpy()
    assert r.last_key_count == want_off[-1]
    start = np.concatenate([[0], np.cumsum(counts)])
    for f in range(len(counts)):
        want, _ = serial(ver[start[f]:start[f + 1]], s['tri'], col[start[f]:start[f + 1]], frames[f])
        assert np.array_equal(out[f], want), f'frame {f} ({counts[f]} meshes)'


def test_random_cases_cover_the_kernel_structure():
    """The seeded cases hold what they claim: each warp kind, boxes of exactly 63, 64 and 65 pixels on both sides of the
    thread / warp split, whole-canvas boxes, every triangle count and canvas, and 1, 3 and 4 channels."""
    seen_kinds, areas, canvases, ntris, chans = set(), set(), set(), set(), set()
    whole = False
    for idx in range(N_CASES):
        s = scene(idx)
        seen_kinds.update(s['kinds'])
        canvases.add((s['h'], s['w']))
        ntris.add(s['tri'].shape[0])
        chans.add(s['c'])
        for m in range(s['ver'].shape[0]):
            b, live = rc.tri_boxes(s['ver'][m], s['tri'], s['h'], s['w'])
            a = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)
            areas.update(a[live].tolist())
            whole |= bool((live & (a == s['h'] * s['w'])).any()) and s['h'] * s['w'] > 64
    assert seen_kinds == set(WARP_KINDS) and {63, 64, 65} <= areas and whole
    assert canvases == set(CANVASES) and ntris == set(NTRI) and chans == {1, 3, 4}


def test_bf16_colours_fail_the_image_check():
    """Negative control: colours rounded to bf16 before drawing must not pass the image comparison of the random cases."""
    failed = 0
    for idx in (3, 4, 10):
        s = scene(idx)
        col16 = torch.from_numpy(s['col']).to(torch.bfloat16).float()
        r = Sim3DR.MeshRenderer(s['tri'], s['ver'].shape[1], DEV)
        img = torch.from_numpy(s['bg'].copy()).to(DEV)
        r.rasterize(img, dev_vertices(s['ver'], s['planar']), col16.to(DEV), reverse=s['reverse'])
        want, _ = serial(s['ver'], s['tri'], s['col'], s['bg'], s['reverse'])
        failed += not np.array_equal(img.cpu().numpy(), want)
    assert failed == 3


# ---- (c) out-of-range values ---------------------------------------------------------------------------------------------------
OOR = rc.out_of_range_cases()


@pytest.mark.parametrize('case', OOR, ids=[c[0] for c in OOR])
def test_out_of_range_values_both_paths(case):
    """A vertex at or beyond 2^31 (or inf / NaN) skips its triangle as in the reference, a colour whose 255 * colour
    reaches 2^31 writes 0, depths at -1e8 / inf / NaN / +-0 and degenerate triangles draw what the serial loop draws --
    on the canvas path (both row orders) and on the frame axis, whose plan boxes follow the same conversions."""
    name, ver, tri, col = case
    h, w = rc.CANVAS
    bg = np.random.default_rng(len(name)).integers(0, 256, (h, w, 3), dtype=np.uint8)
    r = Sim3DR.MeshRenderer(tri, ver.shape[0], DEV)
    for reverse in (False, True):
        img = torch.from_numpy(bg.copy()).to(DEV)
        _, depth = r.rasterize(img, dev_vertices(ver[None], False), torch.from_numpy(col[None]).to(DEV), reverse=reverse,
                               return_depth=True)
        want, dwant = serial(ver[None], tri, col[None], bg, reverse)
        assert np.array_equal(depth.cpu().numpy(), dwant), f'depth, reverse={reverse}'
        assert np.array_equal(img.cpu().numpy(), want), f'image, reverse={reverse}'
    shifted = ver.copy()
    shifted[:, :2] += np.float32([5, 3])
    meshes = np.stack([ver, shifted, ver])
    cols = np.stack([col, col[::-1].copy(), col])
    counts = [1, 0, 2]
    frames = np.stack([bg, bg[::-1].copy(), bg[:, ::-1].copy()])
    v = dev_vertices(meshes, True)
    boxes, key_off = r.plan_frames(v, counts, h, w)
    want_boxes, want_off = plan_want(meshes, tri, counts, h, w)
    assert np.array_equal(boxes.cpu().numpy(), want_boxes), 'plan boxes'
    assert key_off.cpu().numpy().tolist() == want_off.tolist(), 'key offsets'
    out = r.rasterize_frames(torch.from_numpy(frames).to(DEV), v, torch.from_numpy(cols).to(DEV), counts).cpu().numpy()
    assert np.array_equal(out[0], serial(meshes[:1], tri, cols[:1], frames[0])[0]), 'frame 0'
    assert np.array_equal(out[1], frames[1]), 'frame 1 (no mesh)'
    assert np.array_equal(out[2], serial(meshes[1:], tri, cols[1:], frames[2])[0]), 'frame 2'


# ---- (d) normals -----------------------------------------------------------------------------------------------------------------
def normal_case(idx):
    rng = np.random.default_rng(9000 + idx)
    nver = [1, 2, 3, 7, 31, 32, 33, 100, 257, 1000][idx % 10]
    ntri = int(rng.integers(1, 3 * nver + 2))
    tri = rng.integers(0, max(nver - (idx % 3 == 0), 1), (ntri, 3)).astype(np.int32)   # every third case: the last vertex isolated
    b = 1 + idx % 4
    scale = [1.0, 1e3, 1e19, 1e-22][idx % 4]                          # 1e19: cross products overflow; 1e-22: underflow
    ver = (rng.normal(0, 10, (b, nver, 3)) * scale).astype(np.float32)
    if idx % 5 == 1:
        ver = np.round(ver / scale) * np.float32(scale)                # repeated positions: zero-area faces
    if idx % 5 == 2 and ntri > 1:
        tri[::2, 2] = tri[::2, 0]                                     # repeated corners
    if idx % 7 == 3 and nver > 1:
        ver[:, 0, :] = ver[:, 1, :]                                   # a repeated position under two indices
    return ver.astype(np.float32), tri


@pytest.mark.parametrize('idx', range(30))
def test_normals_random_topologies(idx):
    ver, tri = normal_case(idx)
    want = np.stack([rp.get_normal(ver[m], tri) for m in range(ver.shape[0])])
    if rp.have_ref():
        ref = np.stack([rp.get_normal(ver[m], tri, kind='ref') for m in range(ver.shape[0])])
        assert np.array_equal(ref, want, equal_nan=True)
    r = Sim3DR.MeshRenderer(tri, ver.shape[1], DEV)
    for planar in (False, True):
        got = r.normals(dev_vertices(ver, planar)).cpu().numpy()
        assert np.array_equal(got, want, equal_nan=True), f'planar={planar}'


def test_normal_cases_reach_nan_inf_and_isolated_vertices():
    kinds = set()
    for idx in range(30):
        ver, tri = normal_case(idx)
        with np.errstate(all='ignore'):
            n = rp.get_normal(ver[0], tri)
        if np.isnan(n).any():
            kinds.add('nan')
        if len(set(range(ver.shape[1])) - set(tri.ravel().tolist())):
            kinds.add('isolated')
        if (tri[:, 0] == tri[:, 2]).any():
            kinds.add('repeated')
    assert kinds == {'nan', 'isolated', 'repeated'}


# ---- (e) lighting ----------------------------------------------------------------------------------------------------------------
def _cfg(**kw):
    c = dict(RENDER_CFG)
    c.update(kw)
    return c


CFGS = {
    'render': _cfg(),
    'no_ambient': _cfg(intensity_ambient=0.0),
    'no_directional': _cfg(intensity_directional=0.0),
    'no_specular': _cfg(intensity_specular=0.0),
    **{f'exp{e}': _cfg(specular_exp=e) for e in (0, 1, 2, 3, 5, 8)},
    'colours': _cfg(color_ambient=(0.3, 0.6, 0.9), color_directional=(1.0, 0.5, 0.25), intensity_ambient=0.4),
    'defaults': dict(),
}


def light_mesh(name):
    rng = np.random.default_rng(len(name))
    if name.startswith('nver'):
        n = int(name[4:])
        if n == synthetic.NVER:
            ver = np.ascontiguousarray(synthetic.make_render_meshes(1, 120, 120, seed=3)[0].T, np.float32)
            return ver, synthetic.make_render_topology()
        ver = rng.normal(0, 30, (n, 3)).astype(np.float32)
    else:
        ver = rng.normal(0, 30, (300, 3)).astype(np.float32)
        if name == 'negative':
            ver = -np.abs(ver) - 1
        elif name == 'flat':
            ver[:, 1] = 7.0
        elif name == 'equal':
            ver[:] = ver[0]
        elif name == 'nan':
            ver[17, 0] = np.nan
        elif name == 'inf':
            ver[5, 2] = np.inf
        elif name == 'signed_zero':
            ver = np.abs(ver)
            ver[3] = (-0.0, 0.0, -0.0)
            ver[9] = (0.0, -0.0, 0.0)
    n = ver.shape[0]
    tri = rng.integers(0, n, (max(2 * n - 3, 1), 3)).astype(np.int32)
    return ver, tri


MESHES = ['random', 'negative', 'flat', 'equal', 'nan', 'inf', 'signed_zero'] + \
         [f'nver{n}' for n in (1, 255, 257, 16384, 16385, synthetic.NVER)]


def _check_light(got, want, exact, where):
    assert np.array_equal(np.isnan(got), np.isnan(want)), f'{where}: NaN positions'
    if exact:
        assert np.array_equal(got, want, equal_nan=True), f'{where}: {int((got != want).sum())} values differ'
    else:
        ok = ~np.isnan(want)
        assert np.abs(got[ok] - want[ok]).max(initial=0.0) <= LIGHT_TOL, where


@pytest.mark.parametrize('mesh', MESHES)
def test_lighting_configurations(mesh):
    """Bit-exact where the specular term is off; elsewhere within LIGHT_TOL (numpy's powf), NaN positions identical.
    Also the light and the viewer placed exactly on a normalised vertex (a zero-length direction)."""
    ver, tri = light_mesh(mesh)
    with np.errstate(all='ignore'):
        nrm = rp.get_normal(ver, tri)
    r = Sim3DR.MeshRenderer(tri, ver.shape[0], DEV)
    v = dev_vertices(ver[None], MESHES.index(mesh) % 2 == 1)
    nd = torch.from_numpy(nrm[None]).to(DEV)
    with np.errstate(all='ignore'):
        vn = ver - ver.min(0)[None]
        vn /= vn.max()
        vn *= 2
        vn -= vn.max(0)[None] / 2
    cfgs = dict(CFGS)
    k = int(np.argmax(np.isfinite(vn).all(1)))                        # a vertex whose normalised position is finite
    cfgs['light_on_vertex'] = _cfg(light_pos=tuple(float(t) for t in vn[k]))
    cfgs['view_on_vertex'] = _cfg(view_pos=tuple(float(t) for t in vn[k]))
    for name, cfg in cfgs.items():
        with np.errstate(all='ignore'):
            want = rp.lighting(ver, nrm, cfg)
        got = r.colors(v, nd, Sim3DR._light_cfg(**cfg))[0].cpu().numpy()
        spec = cfg.get('intensity_specular', 0.1) > 0 and cfg.get('intensity_directional', 0.6) > 0
        _check_light(got, want, not spec, f'{mesh}/{name}')


@pytest.mark.parametrize('mesh', ['random', 'nan', 'nver257'])
def test_render_pipeline_texture(mesh):
    """The numpy-in ``RenderPipeline`` with a texture: ``texture *= light`` in place, against the numpy restatement."""
    ver, tri = light_mesh(mesh)
    with np.errstate(all='ignore'):
        nrm = rp.get_normal(ver, tri)
    tex0 = np.random.default_rng(1).uniform(0.2, 1.0, ver.shape).astype(np.float32)
    for name in ('render', 'no_specular', 'colours'):
        cfg = CFGS[name]
        tex = tex0.copy()
        bg = np.zeros((16, 16, 3), np.uint8)
        Sim3DR.RenderPipeline(**cfg)(ver, tri, bg, texture=tex)
        with np.errstate(all='ignore'):
            want = tex0 * rp.lighting(ver, nrm, cfg)
        _check_light(tex, want, name != 'render' and name != 'colours', f'{mesh}/{name}')
