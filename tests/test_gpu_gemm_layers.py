"""Every stage of ResNet-50 and of the PointNet heads against the float64 oracle (oracle/gemm64.py), element by element,
and tc_gemm_kernel alone at the shapes and row magnitudes the networks never reach.

Each stage is fed the GPU's own output of the previous stage, so errors do not accumulate and every element is held to
|got - want| <= TAU * S.  Stages that only copy or compare (the max-pools, the face vector, the fp32 bit conversion) and
every row maximum a producer records are compared bit for bit.  The batches put the last 128-row tile of every map size
in each of its shapes (oracle/gemm64.py check_*_batches); the ResNet faces checked include the last face, faces that
straddle the last tile's edge and faces wholly inside it.  H100 only.
"""
import pytest
import torch

from oracle import gemm64, synth_model
from oracle import reference_port as rp
from oracle.stage_check import (HEAD_TOL, TAU, TOL, WIDE, Ratios, check_rowmax, face_picker, make_model, over, report,
                                same_bits, seeded_crops)
from synergynet_b200 import synthetic
from synergynet_b200.backbone import resnet50_conv_keys

pytestmark = pytest.mark.gpu

BARS = TAU['gemm64']
KEYS = resnet50_conv_keys()


# ---- ResNet-50 ------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def rsd():
    return synth_model.build_resnet50_state_dict(0)


@pytest.fixture(scope='module')
def rsd_wide(rsd):
    return synth_model.reparametrize_resnet(rsd, **WIDE['gemm64'])


@pytest.fixture(scope='module')
def rs_model(synth_pack, rsd):
    return make_model(rsd, 'resnet50', strict=False)


@pytest.fixture(scope='module')
def rs_model_wide(synth_pack, rsd_wide):
    return make_model(rsd_wide, 'resnet50', strict=False)


def resnet_ratios(eng, sd, x, faces, ratios):
    """Run every stage of ResNet-50 on batch ``x`` and hold the given faces to the oracle."""
    nf = len(faces)
    pick, where = face_picker(x.shape[0], faces, x.device)

    def run(stage, name):
        out, rm = eng.debug_resnet_until(x, stage)
        if rm is not None:
            check_rowmax(out, rm, name)
        return pick(out)

    stem = run(0, 'stem')
    ratios.add('simt', 'stem', stem, gemm64.resnet_stem(sd, x[faces].cpu()), where(3600))
    pool = run(1, 'maxpool')
    assert same_bits(pool, gemm64.resnet_maxpool(stem, nf)), 'maxpool'

    def conv(i, inp, residual=None):
        got = run(1 + i, KEYS[i][0])
        want = gemm64.resnet_conv(sd, i, inp, nf, residual)
        ratios.add('gemm', KEYS[i][0], got, want, where(got.shape[0] // nf))
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
    ratios.add('pool', 'avgpool', pooled, gemm64.avgpool(X, nf), where(1))
    heads = run(55, 'heads')
    ratios.add('gemm', 'heads', heads, gemm64.resnet_heads(sd, pooled), where(1))
    assert eng.poll_error() == 0


@pytest.mark.parametrize('batch', gemm64.RESNET_BATCHES)
def test_resnet_every_stage_matches_float64_oracle(rs_model, rsd, batch):
    gemm64.check_resnet_batches()
    faces = gemm64.resnet_faces(batch)
    gemm64.check_resnet_faces(batch, faces)
    eng = rs_model._engine(torch.device('cuda', 0))
    ratios = Ratios()
    resnet_ratios(eng, rsd, seeded_crops(batch, 500 + batch), faces, ratios)
    report(f'resnet50 B={batch} faces={faces}', ratios)
    bad = over('gemm64', ratios)
    assert not bad, bad


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
    faces = gemm64.resnet_faces(batch)
    ratios = Ratios()
    resnet_ratios(eng, rsd_wide, seeded_crops(batch, 500 + batch), faces, ratios)
    report(f'resnet50 rescaled B={batch}', ratios)
    bad = over('gemm64', ratios)
    assert not bad, bad


# ---- PointNet heads ---------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def sd_wide(sd):
    return synth_model.reparametrize_pointnet(sd, **WIDE['gemm64'])


@pytest.fixture(scope='module')
def pn_model(synth_pack, sd):
    return make_model(sd)


@pytest.fixture(scope='module')
def pn_model_wide(synth_pack, sd_wide):
    return make_model(sd_wide)


@pytest.fixture(scope='module')
def pn_inputs(synth_pack, sd):
    """Landmarks, avgpool and params of the fp32 port for the largest batch; smaller batches take the first faces."""
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(max(gemm64.POINTNET_BATCHES), seed=71))
    attr, pool = rp.mobilenetv2_forward(sd, x)
    lmk = torch.from_numpy(rp.reconstruct_vertex_62(attr.numpy(), rp.gather_sparse_basis(synthetic.make_3dmm(0))))
    return lmk, pool, attr


def pointnet_ratios(model, sd, lmk, pool, params, ratios):
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
                check_rowmax(out, rm, f'{tag} {name}')
            return out.cpu()

        got = run(0, 'conv1')
        ratios.add('simt', f'{tag} conv1', got, gemm64.pn_conv1(sd, pre, lmk.cpu()), where(68))
        outs = [got]
        for i in range(2, 6):
            got = run(i - 1, f'conv{i}')
            ratios.add('gemm', f'{tag} conv{i}', got, gemm64.pn_conv(sd, pre, f'conv{i}', outs[-1]), where(68))
            outs.append(got)
        glob = run(5, 'global features')
        assert same_bits(glob, gemm64.pn_pool(outs[4])), f'{tag} max-pool'
        if net == 1:
            heads = run(6, 'heads')
            ratios.add('gemm', 'rev heads', heads, gemm64.rev_heads(sd, glob), where(1))
            continue
        fv = run(6, 'face vector')
        assert same_bits(fv, gemm64.face_vector(glob, pool.cpu(), params.cpu())), 'face vector'
        face = run(7, 'conv6 face')
        ratios.add('gemm', 'for conv6 face', face, gemm64.conv6_face(sd, fv), where(1))
        got = run(8, 'conv6 point')
        ratios.add('gemm', 'for conv6 point', got, gemm64.conv6_point(sd, outs[1], face), where(68))
        for i in (7, 8, 9):
            nxt = run(i + 2, f'conv{i}')
            ratios.add('gemm', f'for conv{i}', nxt, gemm64.pn_conv(sd, pre, f'conv{i}', got), where(68))
            got = nxt
        res = run(12, 'residual')
        assert same_bits(res.view(b, 3, 68), gemm64.residual_from_rows(got)), 'point_residual'
    assert eng.poll_error() == 0


@pytest.mark.parametrize('batch', gemm64.POINTNET_BATCHES)
def test_pointnet_every_stage_matches_float64_oracle(pn_model, sd, pn_inputs, batch):
    gemm64.check_pointnet_batches()
    lmk, pool, attr = (t[:batch] for t in pn_inputs)
    ratios = Ratios()
    pointnet_ratios(pn_model, sd, lmk, pool, attr, ratios)
    report(f'pointnet B={batch}', ratios)
    bad = over('gemm64', ratios)
    assert not bad, bad


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
    ratios = Ratios()
    pointnet_ratios(model, sd_wide, lmk, pool, attr, ratios)
    report('pointnet rescaled B=37', ratios)
    bad = over('gemm64', ratios)
    assert not bad, bad


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
    check_rowmax(out, rmo, name)
    if cm is not None:
        m = out_c.shape[0]
        pad_rows = -m % colmax_group
        full = torch.cat([out_c, torch.zeros((pad_rows, out_c.shape[1]))]).view(-1, colmax_group, out_c.shape[1])
        assert same_bits(full.amax(dim=1), cm.cpu().view(torch.float32)), f'colmax {name}'
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
    assert r <= BARS['gemm'], (name, r, ix)


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
    assert r <= BARS['gemm'], (name, r, ix)


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
    assert r <= BARS['gemm'], (r, ix)


def test_wrong_row_scale_fails_the_bar(eng):
    """Negative control: rowmax_in / 8 puts the scaled row max in [2^16, 2^17), past the fp16 range, so the split
    clamps; rowmax_in * 2^24 puts it near 2^-11, so lo falls into the fp16 subnormals.  S comes from the true row
    max.  The bar must flag both by a wide margin."""
    m, k, n = 200, 128, 64
    a = _rows(m, k, seed=23)
    w, bias = _layer(n, k, seed=29)
    true_max = a.abs().amax(dim=1)
    eng.poll_saturation(warn=False)
    r_ok, _ = _kernel_case(eng, a, w, bias, 0, name='true rowmax')
    assert eng.poll_saturation(warn=False) == 0
    r_lo, _ = _kernel_case(eng, a, w, bias, 0, rowmax_in=true_max / 8, name='rowmax / 8')
    assert eng.poll_saturation(warn=False) == 1                    # the split clamped: the flag says so
    r_hi, _ = _kernel_case(eng, a, w, bias, 0, rowmax_in=true_max * 2.0 ** 24, name='rowmax * 2^24')
    assert eng.poll_saturation(warn=False) == 0
    print(f'\n[negative control] true {r_ok:.3e}  rowmax/8 {r_lo:.3e}  rowmax*2^24 {r_hi:.3e}')
    assert r_ok <= BARS['gemm']
    assert r_lo >= 10 * BARS['gemm'] and r_hi >= 10 * BARS['gemm'], (r_lo, r_hi)
