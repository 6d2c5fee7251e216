"""CPU checks of the float64 GEMM-layer oracle, its batch chooser and the rescaled ResNet-50 / PointNet checkpoints used
by tests/test_gpu_gemm_layers.py."""
import pytest
import torch

from oracle import gemm64, synth_model
from oracle import reference_port as rp
from oracle.stage_check import HEAD_TOL, TAU, WIDE
from synergynet_b200 import synthetic
from synergynet_b200.backbone import resnet50_conv_keys

KEYS = resnet50_conv_keys()
NOISE = 2e-6                # fp32 port against the float64 chain, relative to the largest output


@pytest.fixture(scope='module')
def rsd():
    return {'I2P.backbone.' + k: v for k, v in synth_model.build_resnet50_state_dict(0).items()}


@pytest.fixture(scope='module')
def sd():
    return synth_model.build_state_dict(0)


@pytest.fixture(scope='module')
def x3():
    return synthetic.normalize_crops(synthetic.make_structured_crops_u8(3, seed=41))


@pytest.fixture(scope='module')
def heads_in(sd, x3):
    attr, pool = rp.mobilenetv2_forward(sd, x3)
    lmk = torch.from_numpy(rp.reconstruct_vertex_62(attr.numpy(), rp.gather_sparse_basis(synthetic.make_3dmm(0))))
    return lmk, pool, attr


def resnet_chain(sd, x):
    """ResNet-50 stage by stage in float64, every stage fed the previous stage's float64 value."""
    b = x.shape[0]
    stem, _ = gemm64.resnet_stem(sd, x)
    X = gemm64.resnet_maxpool(stem, b).double()
    i = 1
    while i < 53:
        has_ds = i + 3 < 53 and 'downsample' in KEYS[i + 3][0]
        c1, _ = gemm64.resnet_conv(sd, i, X, b)
        c2, _ = gemm64.resnet_conv(sd, i + 1, c1, b)
        ident = gemm64.resnet_conv(sd, i + 3, X, b)[0] if has_ds else X
        X, _ = gemm64.resnet_conv(sd, i + 2, c2, b, ident)
        i += 4 if has_ds else 3
    pooled, _ = gemm64.avgpool(X, b)
    return gemm64.resnet_heads(sd, pooled)[0], pooled


def mlp_chain(sd, lmk, pool, attr):
    """MLP_for and MLP_rev stage by stage in float64 -> (point_residual (B,3,68), MLP_rev output (B,62))."""
    out = {}
    for net, pre in ((0, 'forwardDirection.'), (1, 'reverseDirection.')):
        h, _ = gemm64.pn_conv1(sd, pre, lmk)
        pf = None
        for i in range(2, 6):
            h, _ = gemm64.pn_conv(sd, pre, f'conv{i}', h)
            pf = h if i == 2 else pf
        glob = gemm64.pn_pool(h)
        if net == 1:
            out['rev'] = gemm64.rev_heads(sd, glob)[0]
            continue
        fv = torch.cat([glob, pool.double(), attr.double()[:, 12:62],
                        torch.zeros((glob.shape[0], gemm64.FACE_VEC_LD - 2354), dtype=torch.float64)], 1)
        face, _ = gemm64.conv6_face(sd, fv)
        h, _ = gemm64.conv6_point(sd, pf, face)
        for i in (7, 8, 9):
            h, _ = gemm64.pn_conv(sd, pre, f'conv{i}', h)
        out['res'] = gemm64.residual_from_rows(h)
    return out['res'], out['rev']


def test_resnet_oracle_agrees_with_fp32_reference(rsd, x3):
    want, pooled = rp.resnet50_forward(rsd, x3)
    got, gp = resnet_chain(rsd, x3)
    e, ep = rp.max_rel_err(got.numpy(), want.numpy()), rp.max_rel_err(gp.numpy(), pooled.numpy())
    assert e < NOISE and ep < NOISE, (e, ep)


def test_pointnet_oracle_agrees_with_fp32_reference(sd, heads_in):
    lmk, pool, attr = heads_in
    res, rev = mlp_chain(sd, lmk, pool, attr)
    want_res = rp.mlp_for_forward(sd, lmk, pool, attr[:, 12:52], attr[:, 52:62])
    want_rev = rp.mlp_rev_forward(sd, lmk)
    # the heads amplify a relative perturbation ~50x (tests/test_gpu_heads.py), fp32 rounding included
    e1, e2 = rp.max_rel_err(res.numpy(), want_res.numpy()), rp.max_rel_err(rev.numpy(), want_rev.numpy())
    assert e1 < 50 * NOISE and e2 < 50 * NOISE, (e1, e2)


def test_rescaled_checkpoints_are_exact_and_wide(rsd, sd, x3, heads_in):
    """The reparametrizations compute bit for bit the same fp32 outputs, and they spread the per-channel maxima of the
    hidden tensors they rescale over at least 2^8 inside each row's set of channels."""
    rw = synth_model.reparametrize_resnet(rsd, prefix='I2P.backbone.', **WIDE['gemm64'])
    a0, p0 = rp.resnet50_forward(rsd, x3)
    a1, p1 = rp.resnet50_forward(rw, x3)
    assert torch.equal(a0, a1) and torch.equal(p0, p1)
    f = rw['I2P.backbone.layer3.2.bn1.weight'] / rsd['I2P.backbone.layer3.2.bn1.weight']
    assert float(f.max() / f.min()) == 2.0 ** 10
    assert torch.equal(f, torch.exp2(torch.round(torch.log2(f))))
    lmk, pool, attr = heads_in
    pw = synth_model.reparametrize_pointnet(sd, **WIDE['gemm64'])
    assert torch.equal(rp.mlp_for_forward(sd, lmk, pool, attr[:, 12:52], attr[:, 52:62]),
                       rp.mlp_for_forward(pw, lmk, pool, attr[:, 12:52], attr[:, 52:62]))
    assert torch.equal(rp.mlp_rev_forward(sd, lmk), rp.mlp_rev_forward(pw, lmk))
    h, _ = gemm64.pn_conv1(pw, 'forwardDirection.', lmk)
    for i in range(2, 5):
        h, _ = gemm64.pn_conv(pw, 'forwardDirection.', f'conv{i}', h)
        peak = h.abs().amax(dim=0)
        peak = peak[peak > 0]
        assert float(peak.max() / peak.min()) >= 2 ** 8, i


def test_batch_chooser_covers_every_tile_shape():
    gemm64.check_resnet_batches()
    gemm64.check_pointnet_batches()
    # B = 13 leaves 52 / 109 / 64 / 80 rows in the last tile of the four map sizes, B = 19 76 / 51 / 64 / 48, B = 128 none
    assert [13 * p % 128 for p in gemm64.RESNET_MAPS] == [52, 109, 64, 80]
    assert [19 * p % 128 for p in gemm64.RESNET_MAPS] == [76, 51, 64, 48]
    assert [68 * b % 128 for b in gemm64.POINTNET_BATCHES] == [68, 8, 84, 0]
    with pytest.raises(AssertionError):
        gemm64.check_resnet_batches((13, 128))
    with pytest.raises(AssertionError):
        gemm64.check_pointnet_batches((2, 32))
    for b in gemm64.RESNET_BATCHES:
        faces = gemm64.resnet_faces(b)
        gemm64.check_resnet_faces(b, faces)
        assert len(faces) <= 12
    assert 8 in gemm64.resnet_faces(13)                    # 16-pixel maps: faces 8..12 lie in the last tile (rows 128..207)
    with pytest.raises(AssertionError):
        gemm64.check_resnet_faces(13, [0, 1])


def test_floors_match_the_kernel_scales():
    """eps_row = 2^-2 in the scaled units of a row whose max lands in [2^13, 2^14); eps_n = 2^-2 in those of a weight
    channel whose max lands in [2^8, 2^9)."""
    rm = torch.tensor([1.0, 1.5, 2.0 ** 60, 3.0 * 2.0 ** -60, 0.0])
    assert torch.equal(gemm64.row_floor(rm), torch.tensor([2.0 ** -15, 2.0 ** -15, 2.0 ** 45, 2.0 ** -74, 0.0],
                                                          dtype=torch.float64))
    w = torch.tensor([[0.5, -1.0], [0.0, 0.0], [300.0, 1.0]])
    assert torch.equal(gemm64.chan_floor(w), torch.tensor([2.0 ** -10, 0.0, 2.0 ** -2], dtype=torch.float64))
    # the floors are exact over the whole fp32 range, subnormal maxima included
    rm = torch.tensor([2.0 ** -149, 3.0 * 2.0 ** -140, 2.0 ** -126, 1.5 * 2.0 ** 127])
    assert torch.equal(gemm64.row_floor(rm), torch.exp2(torch.tensor([-164.0, -154.0, -141.0, 112.0], dtype=torch.float64)))
    w = torch.tensor([[2.0 ** -149, 0.0], [-(2.0 ** -130), 2.0 ** -131]])
    assert torch.equal(gemm64.chan_floor(w), torch.exp2(torch.tensor([-159.0, -140.0], dtype=torch.float64)))


def test_check_allows_one_subnormal_spacing_and_infinity_past_the_overflow():
    """|got - want| <= tau * S + 2^-149 at every element, and an infinite result exactly where |want| is within tau * S
    of the fp32 overflow threshold or past it."""
    from oracle.check64 import F32_OVERFLOW, ratio
    tau = TAU['gemm64']['gemm']
    want = torch.tensor([0.0, 2.0 ** -150, 1.0, 2.0 ** 129, -(2.0 ** 129), F32_OVERFLOW - 2.0 ** 100, 2.0 ** 127],
                        dtype=torch.float64)
    s = torch.tensor([0.0, 0.0, 1.0, 2.0 ** 100, 2.0 ** 100, 2.0 ** 100 / tau, 1.0], dtype=torch.float64)
    got = torch.tensor([2.0 ** -149, 0.0, 1.0 + 2 * tau, float('inf'), -float('inf'), float('inf'), float('inf')])
    r = ratio(got, want, s)
    assert r[0] == 0 and r[1] == 0                       # one subnormal spacing off, with S = 0
    assert r[2] > tau                                     # 2 tau * S off
    assert r[3] == 0 and r[4] == 0                        # past the threshold: Inf with the sign of want
    assert r[5] <= tau                                    # within tau * S of it
    assert r[6] > 1e30                                    # 2^127 is finite in fp32: Inf is far off
    assert ratio(-got[3:4], want[3:4], s[3:4])[0] == float('inf')   # the wrong infinity
    assert ratio(torch.tensor([3e38]), want[3:4], s[3:4])[0] > 1e6  # a finite result past the overflow


def test_checker_flags_a_small_channel_that_max_rel_err_misses(sd, heads_in):
    """A channel of conv5's output (rescaled MLP_for) whose values are 1-10 % of the tensor's maximum, scaled by
    1 + 1e-3: the per-element check flags it, while max_rel_err under HEAD_TOL passes the same tensor."""
    lmk, pool, attr = heads_in
    pw = synth_model.reparametrize_pointnet(sd, **WIDE['gemm64'])
    pre = 'forwardDirection.'
    h, _ = gemm64.pn_conv1(pw, pre, lmk)
    for i in range(2, 5):
        h, _ = gemm64.pn_conv(pw, pre, f'conv{i}', h)
    want, s = gemm64.pn_conv(pw, pre, 'conv5', h)
    peak = want.abs().amax(dim=0)
    small = ((peak > 0.01 * peak.max()) & (peak < 0.1 * peak.max())).nonzero().flatten()
    assert len(small) > 0
    c = int(small[0])
    bad = want.clone()
    bad[:, c] *= 1 + 1e-3
    assert rp.max_rel_err(bad.numpy(), want.numpy()) < HEAD_TOL
    r, where = gemm64.worst(bad, want, s)
    assert r > 10 * TAU['gemm64']['gemm'] and where[1] == c, (r, where)
    assert gemm64.worst(want.float(), want, s)[0] < TAU['gemm64']['gemm']
