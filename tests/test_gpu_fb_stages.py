"""Every launch of the FaceBoxes detector network against the float64 oracle (oracle/fb64.py), element by element, at
image sizes that put the last 64-row tile of every map the conv kernel tiles in each of its shapes (fb64.check_sizes).

Each stage is fed the GPU's own output of the stages before it (``FaceBoxesNet.debug_forward_until``), so errors do not
accumulate and every element is held to |got - want| <= TAU * S.  The max-pools are compared bit for bit.  Every
inception branch and every head must write its slice of the shared tensor and nothing else.  H100 only.
"""
import pytest
import torch

from oracle import fb64
from oracle.stage_check import TAU, Ratios, over, report, same_bits
from synergynet_b200 import faceboxes, synthetic

pytestmark = pytest.mark.gpu

BARS = TAU['fb64']
NONZERO = 0.25              # every ReLU stage: the float64 chain measures 37-69 % nonzero on these scenes at every size
SIZES = fb64.choose_sizes()


def _name(i):
    st = fb64.STAGES[i]
    return f'{i} {fb64.LAYERS[st.layer].name}' if st.layer is not None else f'{i} {st.kind}'


@pytest.fixture(scope='module')
def sd():
    return synthetic.make_faceboxes_state_dict(0)


@pytest.fixture(scope='module')
def net(sd):
    return faceboxes.FaceBoxesNet(sd, torch.device('cuda', 0))


def _scene(h, w):
    return torch.from_numpy(synthetic.make_scene_u8(h, w, h * 7 + w)).cuda()


def run_stages(net, img):
    """Every stage's destination tensor, stopping after each launch in production order (on the CPU)."""
    got = {i: net.debug_forward_until(img, i).cpu() for i in range(len(fb64.STAGES))}
    torch.cuda.synchronize()
    return got


def stage_ratios(sd, img, got, ratios):
    """Hold every stage to the oracle on the GPU's own inputs: rounding stages into ``ratios``, max-pools bit for bit.
    Returns the fraction of nonzero elements of every ReLU stage."""
    h, w = int(img.shape[0]), int(img.shape[1])
    image = img.cpu()
    nonzero = {}
    for i, st in enumerate(fb64.STAGES):
        r = fb64.stage(sd, i, [image if s == 'image' else got[s] for s in st.inputs])
        part = fb64.owned(i, got[i], h, w)
        if st.kind == 'maxpool':
            assert same_bits(part, r), f'{(h, w)} {_name(i)}'
            continue
        ratios.add(st.kind, _name(i), part, r)
        if st.kind == 'conv' and fb64.LAYERS[st.layer].act:
            nonzero[i] = float((part != 0).double().mean())
    return nonzero


def check_slices(got, h, w):
    """Each inception branch and each head writes its slice of the shared tensor and leaves every other element as the
    launch before it left it; after the last one the tensor is the slices each returned at its own stop."""
    for b, last in enumerate(fb64.BLOCK_LAST):
        writers = [s for s in range(last - 7, last + 1) if fb64.STAGES[s].dest == fb64.STAGES[last].dest]
        # what the block output buffer held before the block's first branch: nothing known (inception1), the max-pool
        # output (inception2 writes into that buffer) or inception1's output (inception3 writes into that one)
        before = (None, got[3], got[fb64.BLOCK_LAST[0]])[b]
        for s in writers:
            lo, hi = fb64.STAGES[s].owns
            keep = torch.ones(128, dtype=torch.bool)
            keep[lo:hi] = False
            if before is not None:
                assert same_bits(got[s][..., keep], before[..., keep]), f'{(h, w)} {_name(s)} wrote outside {lo}..{hi}'
            assert same_bits(got[last][..., lo:hi], got[s][..., lo:hi]), f'{(h, w)} block {b + 1} slice {lo}..{hi}'
            before = got[s]
    for head, last in fb64.HEAD_LAST.items():
        before = None
        for s in range(last - 2, last + 1):
            e0, e1 = fb64.head_range(s, h, w)
            t = got[s]
            assert same_bits(got[last][e0:e1], t[e0:e1]), f'{(h, w)} {head} head {_name(s)}'
            assert not torch.isnan(t[e0:e1]).any(), f'{(h, w)} {_name(s)} left part of its slice unwritten'
            assert torch.isnan(t[e1:]).all(), f'{(h, w)} {_name(s)} wrote past its slice'
            if before is not None:
                assert same_bits(t[:e0], before[:e0]), f'{(h, w)} {_name(s)} wrote before its slice'
            before = t


@pytest.mark.parametrize('hw', SIZES, ids=[f'{h}x{w}' for h, w in SIZES])
def test_every_stage_matches_float64_oracle(sd, net, hw):
    fb64.check_sizes(SIZES)
    h, w = hw
    img = _scene(h, w)
    got = run_stages(net, img)
    ratios = Ratios()
    nonzero = stage_ratios(sd, img, got, ratios)
    report(f'faceboxes {h}x{w}', ratios)
    bad = over('fb64', ratios)
    assert not bad, bad
    check_slices(got, h, w)
    low = {_name(i): f for i, f in nonzero.items() if f < NONZERO}
    assert not low, low
    loc, conf = net.forward(img)                        # the debug stops run the production sequence
    torch.cuda.synchronize()
    assert same_bits(loc.cpu().reshape(-1), got[fb64.HEAD_LAST['loc']])
    assert same_bits(conf.cpu().reshape(-1), got[len(fb64.STAGES) - 1])


def test_workspace_reallocation_keeps_results(sd):
    """One handle runs every size in turn (each change of size reallocates its workspace), then the first size again."""
    net = faceboxes.FaceBoxesNet(sd, torch.device('cuda', 0))
    first = None
    for h, w in SIZES:
        loc, conf = net.forward(_scene(h, w))
        torch.cuda.synchronize()
        if first is None:
            first = (loc.cpu(), conf.cpu())
    loc, conf = net.forward(_scene(*SIZES[0]))
    torch.cuda.synchronize()
    assert same_bits(loc.cpu(), first[0]) and same_bits(conf.cpu(), first[1])
    net.close()


def test_debug_entry_errors(net):
    """A wrong out_numel is SYN_ERR_SHAPE, an uncommitted handle SYN_ERR_STATE, a null output SYN_ERR_INVALID."""
    import ctypes as C
    from synergynet_b200 import _lib
    lib = _lib.load()
    h, w = fb64.GOLDEN[1]
    img = _scene(h, w)
    loc, conf = torch.empty(4 * fb64.num_priors(h, w), device='cuda'), torch.empty(2 * fb64.num_priors(h, w), device='cuda')
    out = torch.empty(faceboxes.debug_stage_shape(5, h, w), device='cuda')
    args = lambda stage, o, n, hd=net._h: (hd, img.data_ptr(), h, w, stage, o, n, loc.data_ptr(), conf.data_ptr(), None)
    assert lib.syn_fb_debug_forward_until(*args(5, out.data_ptr(), out.numel())) == 0
    assert lib.syn_fb_debug_forward_until(*args(5, out.data_ptr(), out.numel() - 1)) == 4
    assert lib.syn_fb_debug_forward_until(*args(5, None, out.numel())) == 1
    fresh = C.c_void_p()
    _lib.check(lib.syn_fb_create(0, C.byref(fresh)))
    assert lib.syn_fb_debug_forward_until(*args(5, out.data_ptr(), out.numel(), fresh)) == 3
    lib.syn_fb_destroy(fresh)
    torch.cuda.synchronize()


def test_bf16_weights_fail_the_bar(sd):
    """Negative control: a handle whose conv weights were rounded to bf16 before upload, held to the oracle of the unrounded
    weights, must exceed TAU at every conv stage and reach 10x TAU at its worst."""
    bad = dict(sd)
    for L in fb64.LAYERS:
        key = f'{L.name}.conv.weight' if L.bn else f'{L.name}.weight'
        bad[key] = sd[key].to(torch.bfloat16).float()
    net = faceboxes.FaceBoxesNet(bad, torch.device('cuda', 0))
    h, w = fb64.GOLDEN[0]
    img = _scene(h, w)
    ratios = Ratios()
    stage_ratios(sd, img, run_stages(net, img), ratios)
    conv = {s: v[0] for s, v in ratios.items() if v[2] == 'conv'}
    lo, hi = min(conv, key=conv.get), max(conv, key=conv.get)
    print(f'\n[bf16 weights] smallest {conv[lo]:.3e} at {lo}, largest {conv[hi]:.3e} at {hi}')
    assert conv[lo] > BARS['conv'] and conv[hi] >= 10 * BARS['conv'], conv
    net.close()
