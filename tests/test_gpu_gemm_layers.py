"""Every stage of ResNet-50 and of the PointNet heads against the float64 oracle (oracle/gemm64.py), element by element,
and tc_gemm_kernel alone at the shapes and row magnitudes the networks never reach.

Each stage is fed the GPU's own output of the previous stage, so errors do not accumulate and every element is held to
|got - want| <= TAU * S.  Stages that only copy or compare (the max-pools, the face vector, the fp32 bit conversion) and
every row maximum a producer records are compared bit for bit.  The batches put the last 128-row tile of every map size
in each of its shapes (oracle/gemm64.py check_*_batches); the ResNet faces checked include the last face, faces that
straddle the last tile's edge and faces wholly inside it.  H100 only.
"""
import types

import pytest
import torch

from oracle import gemm64, synth_model
from oracle import reference_port as rp
from synergynet_b200 import synthetic
from synergynet_b200.backbone import resnet50_conv_keys

pytestmark = pytest.mark.gpu

# The bar: |got - want| <= TAU * S at every element, per stage kind, at most 4x the worst ratio measured on an H100
# 80GB HBM3 (132 SMs, 700 W power limit) over the batches, both checkpoints and the kernel-level cases of this file
# (worst in the comment):
TAU = {'gemm': 8e-6,        # 3.13e-06: tc_gemm_kernel, ResNet layer4.0.conv2 (K = 4608) at B = 19; PointNet 1.67e-06
       'simt': 2e-6,        # 7.18e-07: fp32 CUDA cores, ResNet stem (K = 147); PointNet conv1 9.96e-08
       'pool': 8e-7}        # 2.39e-07: fp32 average pool
# The ratio grows with K (the fp32 accumulation over k): 1.98e-06 for K = 2360, 2.52e-06 for a 3x3 conv with K = 2304.
# Negative control: rowmax_in / 8 measures 2.21e-01 and rowmax_in * 2^24 2.13e-04, >= 26x the bar.
WIDE = dict(seed=11, lo=-6, hi=4)         # hidden-channel factors 2^-6 .. 2^4
TOL = 1e-4
HEAD_TOL = 3e-4                           # tests/test_gpu_heads.py
KEYS = resnet50_conv_keys()


class Worst:
    """Largest ratio per stage kind, with where it occurred."""

    def __init__(self):
        self.by_kind = {}

    def add(self, kind, stage, got, want_s, where_fn=lambda ix: ix):
        r, ix = gemm64.worst(got, *want_s)
        if r >= self.by_kind.get(kind, (-1.0,))[0]:
            self.by_kind[kind] = (r, stage, where_fn(ix))
        return r

    def over(self):
        return {k: v for k, v in self.by_kind.items() if v[0] > TAU[k]}

    def report(self, tag):
        print(f'\n[{tag}] ' + '  '.join(f'{k}: {r:.3e} at {s} {w}' for k, (r, s, w) in self.by_kind.items()))


def _same_bits(a, b):
    return torch.equal(a.float().contiguous().view(torch.int32), b.float().contiguous().view(torch.int32))


def _check_rowmax(out, rm, stage):
    assert rm is not None and torch.equal(rm, gemm64.rowmax_bits(out)), f'rowmax of {stage}'


# ---- ResNet-50 ------------------------------------------------------------------------------------------------------

def _resnet_model(sd):
    from synergynet_b200 import model_building
    m = model_building.SynergyNet(types.SimpleNamespace(arch='resnet50', img_size=120, devices_id=[0]))
    m.load_state_dict({'I2P.backbone.' + k: v for k, v in sd.items()}, strict=False)
    return m.eval()


@pytest.fixture(scope='module')
def rsd():
    return synth_model.build_resnet50_state_dict(0)


@pytest.fixture(scope='module')
def rsd_wide(rsd):
    return synth_model.reparametrize_resnet(rsd, **WIDE)


@pytest.fixture(scope='module')
def rs_model(synth_pack, rsd):
    return _resnet_model(rsd)


@pytest.fixture(scope='module')
def rs_model_wide(synth_pack, rsd_wide):
    return _resnet_model(rsd_wide)


def resnet_ratios(eng, sd, x, faces, worst):
    """Run every stage of ResNet-50 on batch ``x`` and hold the given faces to the oracle."""
    b, nf = x.shape[0], len(faces)
    fidx = torch.tensor(faces, device=x.device)
    pick = lambda t: t.view(b, -1, t.shape[1]).index_select(0, fidx).reshape(-1, t.shape[1]).cpu()

    def where(per_face):
        return lambda ix: (faces[ix[0] // per_face], ix[0] % per_face, ix[1])

    def run(stage, name):
        out, rm = eng.debug_resnet_until(x, stage)
        if rm is not None:
            _check_rowmax(out, rm, name)
        return pick(out)

    stem = run(0, 'stem')
    worst.add('simt', 'stem', stem, gemm64.resnet_stem(sd, x.index_select(0, fidx).cpu()), where(3600))
    pool = run(1, 'maxpool')
    assert _same_bits(pool, gemm64.resnet_maxpool(stem, nf)), 'maxpool'

    def conv(i, inp, residual=None):
        got = run(1 + i, KEYS[i][0])
        want = gemm64.resnet_conv(sd, i, inp, nf, residual)
        worst.add('gemm', KEYS[i][0], got, want, where(got.shape[0] // nf))
        return got

    X, i = pool, 1
    while i < 53:
        has_ds = i + 3 < 53 and 'downsample' in KEYS[i + 3][0]
        c1 = conv(i, X)
        c2 = conv(i + 1, c1)
        ident = conv(i + 3, X) if has_ds else X
        X = conv(i + 2, c2, ident)
        i += 4 if has_ds else 3
    pooled = run(54, 'avgpool')
    worst.add('pool', 'avgpool', pooled, gemm64.avgpool(X, nf), where(1))
    heads = run(55, 'heads')
    worst.add('gemm', 'heads', heads, gemm64.resnet_heads(sd, pooled), where(1))
    assert eng.poll_error() == 0


def _crops(batch, seed):
    return synthetic.normalize_crops(synthetic.make_structured_crops_u8(batch, seed=seed)).cuda()


@pytest.mark.parametrize('batch', gemm64.RESNET_BATCHES)
def test_resnet_every_stage_matches_float64_oracle(rs_model, rsd, batch):
    gemm64.check_resnet_batches()
    faces = gemm64.resnet_faces(batch)
    gemm64.check_resnet_faces(batch, faces)
    eng = rs_model._engine(torch.device('cuda', 0))
    w = Worst()
    resnet_ratios(eng, rsd, _crops(batch, 500 + batch), faces, w)
    w.report(f'resnet50 B={batch} faces={faces}')
    assert not w.over(), w.over()


def test_resnet_rescaled_checkpoint(rs_model_wide, rsd_wide):
    """The rescaled checkpoint computes the same function (out102 of the reference module within 1e-4) and holds every
    stage to the same bar with hidden channels spread over 2^10."""
    from golden.vectors import load_ref_vectors
    gold = load_ref_vectors()
    eng = rs_model_wide._engine(torch.device('cuda', 0))
    out, _ = eng.forward_resnet50(synthetic.normalize_crops(torch.from_numpy(gold['x_u8']))[:4].cuda())
    err = rp.max_rel_err(out.cpu().numpy(), gold['resnet50_out102'])
    print(f'\n[resnet50 rescaled] out102 err {err:.3e}')
    assert err < TOL
    batch = gemm64.RESNET_BATCHES[0]
    w = Worst()
    resnet_ratios(eng, rsd_wide, _crops(batch, 500 + batch), gemm64.resnet_faces(batch), w)
    w.report(f'resnet50 rescaled B={batch}')
    assert not w.over(), w.over()


# ---- PointNet heads ---------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def sd_wide(sd):
    return synth_model.reparametrize_pointnet(sd, **WIDE)


@pytest.fixture(scope='module')
def pn_model(synth_pack, sd):
    return _mobilenet_model(sd)


@pytest.fixture(scope='module')
def pn_model_wide(synth_pack, sd_wide):
    return _mobilenet_model(sd_wide)


@pytest.fixture(scope='module')
def pn_inputs(synth_pack, sd):
    """Landmarks, avgpool and params of the fp32 port for the largest batch; smaller batches take the first faces."""
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(max(gemm64.POINTNET_BATCHES), seed=71))
    attr, pool = rp.mobilenetv2_forward(sd, x)
    lmk = torch.from_numpy(rp.reconstruct_vertex_62(attr.numpy(), rp.gather_sparse_basis(synthetic.make_3dmm(0))))
    return lmk, pool, attr


def _mobilenet_model(sd):
    from synergynet_b200 import model_building
    m = model_building.SynergyNet(types.SimpleNamespace(arch='mobilenet_v2', img_size=120, devices_id=[0]))
    m.load_state_dict(sd, strict=True)
    return m.eval()


def pointnet_ratios(model, sd, lmk, pool, params, worst):
    b = lmk.shape[0]
    lmk, pool, params = lmk.cuda(), pool.cuda(), params.cuda()
    eng = model._pointnet_engine(lmk, 0)                  # hands both heads' weights to the engine
    assert model._pointnet_engine(lmk, 1) is eng
    where = lambda per_face: (lambda ix: (ix[0] // per_face, ix[0] % per_face, ix[1]))
    for net, pre in ((0, 'forwardDirection.'), (1, 'reverseDirection.')):
        tag = 'for' if net == 0 else 'rev'

        def run(stage, name):
            out, rm = eng.debug_pointnet_until(net, lmk, stage, pool, params)
            if rm is not None:
                _check_rowmax(out, rm, f'{tag} {name}')
            return out.cpu()

        got = run(0, 'conv1')
        worst.add('simt', f'{tag} conv1', got, gemm64.pn_conv1(sd, pre, lmk.cpu()), where(68))
        outs = [got]
        for i in range(2, 6):
            got = run(i - 1, f'conv{i}')
            worst.add('gemm', f'{tag} conv{i}', got, gemm64.pn_conv(sd, pre, f'conv{i}', outs[-1]), where(68))
            outs.append(got)
        glob = run(5, 'global features')
        assert _same_bits(glob, gemm64.pn_pool(outs[4])), f'{tag} max-pool'
        if net == 1:
            heads = run(6, 'heads')
            worst.add('gemm', 'rev heads', heads, gemm64.rev_heads(sd, glob), where(1))
            continue
        fv = run(6, 'face vector')
        assert _same_bits(fv, gemm64.face_vector(glob, pool.cpu(), params.cpu())), 'face vector'
        face = run(7, 'conv6 face')
        worst.add('gemm', 'for conv6 face', face, gemm64.conv6_face(sd, fv), where(1))
        got = run(8, 'conv6 point')
        worst.add('gemm', 'for conv6 point', got, gemm64.conv6_point(sd, outs[1], face), where(68))
        for i in (7, 8, 9):
            nxt = run(i + 2, f'conv{i}')
            worst.add('gemm', f'for conv{i}', nxt, gemm64.pn_conv(sd, pre, f'conv{i}', got), where(68))
            got = nxt
        res = run(12, 'residual')
        assert _same_bits(res.view(b, 3, 68), gemm64.residual_from_rows(got)), 'point_residual'
    assert eng.poll_error() == 0


@pytest.mark.parametrize('batch', gemm64.POINTNET_BATCHES)
def test_pointnet_every_stage_matches_float64_oracle(pn_model, sd, pn_inputs, batch):
    gemm64.check_pointnet_batches()
    lmk, pool, attr = (t[:batch] for t in pn_inputs)
    w = Worst()
    pointnet_ratios(pn_model, sd, lmk, pool, attr, w)
    w.report(f'pointnet B={batch}')
    assert not w.over(), w.over()


def test_pointnet_rescaled_checkpoint(pn_model_wide, sd_wide, pn_inputs):
    """The rescaled heads compute the same function: the reference's losses, point_residual and MLP_rev output within
    HEAD_TOL, and every stage under the same bar."""
    from golden.vectors import load_ref_vectors
    gold = load_ref_vectors()
    model = pn_model_wide
    x = synthetic.normalize_crops(torch.from_numpy(gold['x_u8'])).cuda()
    loss = model(x, torch.from_numpy(gold['fwd_target']).cuda())
    for k, v in loss.items():
        assert rp.max_rel_err(v.cpu().numpy(), gold['fwd_' + k]) < HEAD_TOL, k
    t = model.last_forward
    assert rp.max_rel_err(t['point_residual'].cpu().numpy(), gold['fwd_point_residual']) < HEAD_TOL
    assert rp.max_rel_err(t['_3D_attr_S2'].cpu().numpy(), gold['fwd_3D_attr_S2']) < HEAD_TOL
    lmk, pool, attr = (t[:37] for t in pn_inputs)
    w = Worst()
    pointnet_ratios(model, sd_wide, lmk, pool, attr, w)
    w.report('pointnet rescaled B=37')
    assert not w.over(), w.over()


# ---- tc_gemm_kernel alone ---------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def eng(pn_model):
    return pn_model._engine(torch.device('cuda', 0))


def _rows(m, k, seed, spread=True):
    """Rows of mixed sign whose columns spread over 2^-6 .. 2^4 (as the rescaled checkpoints' activations do)."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn((m, k), generator=g)
    if spread:
        a *= torch.exp2(torch.randint(-6, 5, (k,), generator=g).float())
    return a


def _layer(n, k, seed):
    g = torch.Generator().manual_seed(seed + 1)
    w = torch.randn((n, k), generator=g) / k ** 0.5 * torch.exp2(torch.randint(-4, 3, (n, 1), generator=g).float())
    return w, torch.randn((n,), generator=g)


def _kernel_case(eng, a, w, bias, act, rowmax_in=None, conv=None, residual=None, addend=None, addend_group=1,
                 colmax_group=0, name=''):
    """One syn_debug_gemm launch checked against the oracle: returns the worst ratio; rowmax_out (and colmax) exact."""
    if conv is None:
        rows = a
        true_max = a.abs().amax(dim=1)
    else:
        ks, st, pad, ho, wo = conv
        rows = gemm64.patches(a, ks, st, pad)
        true_max = a.abs().amax(dim=3).reshape(-1)                     # per input pixel
    if rowmax_in is None:
        rowmax_in = true_max
    out, rmo, cm = eng.debug_gemm(w, bias, a, rowmax_in.float().view(torch.int32), act=act, conv=conv,
                                  residual=residual, addend=addend, addend_group=addend_group, colmax_group=colmax_group)
    add = None if addend is None else addend.repeat_interleave(addend_group, dim=0)[:rows.shape[0]]
    want = gemm64.gemm(rows, w, bias, act == 2, addend=add, residual=residual)
    out_c = out.cpu()
    _check_rowmax(out, rmo, name)
    if cm is not None:
        m = out_c.shape[0]
        pad_rows = -m % colmax_group
        full = torch.cat([out_c, torch.zeros((pad_rows, out_c.shape[1]))]).view(-1, colmax_group, out_c.shape[1])
        assert _same_bits(full.amax(dim=1), cm.cpu().view(torch.float32)), f'colmax {name}'
    return gemm64.worst(out_c, *want)


GEMM_CASES = (
    # (name, M, K, N, act, extras): plain rows; M around the 64/128-row edges, every N-range width, a kc = 16 tail
    [(f'N{n}', 193, 72, n, 2, {}) for n in (3, 16, 48, 62, 102, 256, 257, 1000)] +
    [(f'M{m}', m, 64, 64, 0, {}) for m in (1, 63, 64, 65, 127, 128, 129, 191, 192, 256)] +
    [(f'K{k}', 129, k, 62, 2, {}) for k in (8, 16, 40, 48, 2360)] +
    [('residual', 150, 96, 80, 2, {'residual': True}), ('addend', 340, 64, 48, 2, {'addend': 68})] +
    [(f'colmax{g}', 400, 64, 48, 2, {'colmax': g}) for g in (5, 16, 68, 200)])


@pytest.mark.parametrize('case', GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_gemm_kernel_shapes(eng, case):
    name, m, k, n, act, ex = case
    a = _rows(m, k, seed=m * 7 + k)
    w, bias = _layer(n, k, seed=n)
    res = torch.randn((m, n), generator=torch.Generator().manual_seed(3)) if ex.get('residual') else None
    add = None
    if 'addend' in ex:
        add = torch.randn((-(-m // ex['addend']), n), generator=torch.Generator().manual_seed(4)) * 4
    r, ix = _kernel_case(eng, a, w, bias, act, residual=res, addend=add, addend_group=ex.get('addend', 1),
                         colmax_group=ex.get('colmax', 0), name=name)
    print(f'\n[gemm {name}] worst {r:.3e} at {ix}')
    assert r <= TAU['gemm'], (name, r, ix)


CONV_CASES = (   # (name, B, H, W, C, N, ksize, stride, pad, residual)
    ('3x3s1_7x5', 3, 7, 5, 16, 24, 3, 1, 1, False),
    ('3x3s2_15x15', 2, 15, 15, 8, 40, 3, 2, 1, True),
    ('3x3s2_30x30', 1, 30, 30, 64, 64, 3, 2, 1, False),
    ('1x1s2_8x8', 4, 8, 8, 32, 64, 1, 2, 0, False),
    ('3x3s1_4x4', 5, 4, 4, 256, 256, 3, 1, 1, True),
)


@pytest.mark.parametrize('case', CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_gemm_kernel_conv_mode(eng, case):
    name, b, h, wd, c, n, ks, st, pad, with_res = case
    ho, wo = (h + 2 * pad - ks) // st + 1, (wd + 2 * pad - ks) // st + 1
    a = _rows(b * h * wd, c, seed=h * 31 + c).clamp_min(0).view(b, h, wd, c)     # ReLU maps, as the network feeds
    w, bias = _layer(n, ks * ks * c, seed=n + ks)
    res = torch.randn((b * ho * wo, n), generator=torch.Generator().manual_seed(5)) if with_res else None
    r, ix = _kernel_case(eng, a, w, bias, 2, conv=(ks, st, pad, ho, wo), residual=res, name=name)
    print(f'\n[gemm conv {name}] worst {r:.3e} at {ix}')
    assert r <= TAU['gemm'], (name, r, ix)


def test_gemm_kernel_row_magnitudes(eng):
    """Rows whose max is 2^60 or 2^-60, all-zero rows, and rows where one element is 2^20 times all the others: the
    row scale keeps each of them exact to the same bar (no bias, so nothing masks a wrong small row)."""
    m, k, n = 160, 96, 72
    a = _rows(m, k, seed=17, spread=False)
    a[0:16] *= 2.0 ** 60
    a[16:32] *= 2.0 ** -60
    a[32:48] = 0.0
    a[48:64] *= 2.0 ** -20
    a[48:64, 5] = 1.0 + torch.arange(16) / 16.0
    a[130:140] = 0.0                                                          # zero rows in warpgroup 0 of the last tile
    w, _ = _layer(n, k, seed=9)
    r, ix = _kernel_case(eng, a, w, torch.zeros(n), 0, name='magnitudes')
    print(f'\n[gemm row magnitudes] worst {r:.3e} at {ix}')
    assert r <= TAU['gemm'], (r, ix)


def test_wrong_row_scale_fails_the_bar(eng):
    """Negative control: rowmax_in / 8 puts the scaled row max in [2^16, 2^17), past the fp16 range, so the split
    clamps; rowmax_in * 2^24 puts it near 2^-11, so lo falls into the fp16 subnormals.  S comes from the true row
    max.  The bar must flag both by a wide margin."""
    m, k, n = 200, 128, 64
    a = _rows(m, k, seed=23)
    w, bias = _layer(n, k, seed=29)
    true_max = a.abs().amax(dim=1)
    r_ok, _ = _kernel_case(eng, a, w, bias, 0, name='true rowmax')
    r_lo, _ = _kernel_case(eng, a, w, bias, 0, rowmax_in=true_max / 8, name='rowmax / 8')
    r_hi, _ = _kernel_case(eng, a, w, bias, 0, rowmax_in=true_max * 2.0 ** 24, name='rowmax * 2^24')
    print(f'\n[negative control] true {r_ok:.3e}  rowmax/8 {r_lo:.3e}  rowmax*2^24 {r_hi:.3e}')
    assert r_ok <= TAU['gemm']
    assert r_lo >= 10 * TAU['gemm'] and r_hi >= 10 * TAU['gemm'], (r_lo, r_hi)
