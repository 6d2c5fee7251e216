"""Float64 per-stage oracle of the FaceBoxes detector network (reference FaceBoxes/models/faceboxes.py:8-150), with a
per-element error scale, the table of its 39 launches and the image sizes that put its kernels' edges under a check.
TEST INFRASTRUCTURE.

The contract is that of ``block64.py`` / ``gemm64.py``: every stage is fed the exact fp32 tensor the GPU stage was fed
(the GPU's own output of the stages before it, as ``FaceBoxesNet.debug_forward_until`` returns them) and returns
``(want, S)``; a stage passes when |got - want| <= tau * S at every element (``check64.worst``).  BatchNorm is folded
here, in float64, from the reference-schema state dict (``check64.fold_bn``), not from the library's folded weights.

Every convolution runs on CUDA cores in fp32 FMA (``fb_conv_kernel``, ``fb_conv_smalln_kernel``, csrc/kernels_detect.cuh),
so S = sum_k |a_k||w_k| + |b| (``gemm64.simt``).  conv1's operand is u8 - mean, exact in fp32.  CReLU writes relu(v) to
channel c and relu(-v) to channel c + cout; both carry the S of v.  The average pool sums nine taps in fp32 and divides
by 9 at every pixel (count_include_pad), so S = sum |x| / 9 over the in-bounds taps.  The max-pools do not round and
are compared bit for bit.  The softmax of the GPU's own logits rounds a - max(a, b) before expf, an absolute error in
the exponent, then divides: S = p (1 + |a - b|).
"""
from __future__ import annotations

from collections import namedtuple
from typing import Callable, Dict, List, Tuple

import torch
import torch.nn.functional as F

from oracle import gemm64
from oracle.check64 import Pair, fold_bn, strip_prefix

MEAN_BGR = (104.0, 117.0, 123.0)                 # FaceBoxes.py:92
FB_BM = 64                                       # output pixels per CTA of fb_conv_kernel

# ---- the network -------------------------------------------------------------------------------------------------------

Layer = namedtuple('Layer', 'name cin cout k stride pad bn act')       # act: 0 linear, 1 ReLU, 2 CReLU (2 * cout outputs)


def _layers() -> List[Layer]:
    out = [Layer('conv1', 3, 24, 7, 4, 3, True, 2), Layer('conv2', 48, 64, 5, 2, 2, True, 2)]      # faceboxes.py:68-72
    for b in (1, 2, 3):                                                                             # Inception :21-47
        p = f'inception{b}.'
        out += [Layer(p + 'branch1x1', 128, 32, 1, 1, 0, True, 1), Layer(p + 'branch1x1_2', 128, 32, 1, 1, 0, True, 1),
                Layer(p + 'branch3x3_reduce', 128, 24, 1, 1, 0, True, 1), Layer(p + 'branch3x3', 24, 32, 3, 1, 1, True, 1),
                Layer(p + 'branch3x3_reduce_2', 128, 24, 1, 1, 0, True, 1),
                Layer(p + 'branch3x3_2', 24, 32, 3, 1, 1, True, 1), Layer(p + 'branch3x3_3', 32, 32, 3, 1, 1, True, 1)]
    out += [Layer('conv3_1', 128, 128, 1, 1, 0, True, 1), Layer('conv3_2', 128, 256, 3, 2, 1, True, 1),   # :78-82
            Layer('conv4_1', 256, 128, 1, 1, 0, True, 1), Layer('conv4_2', 128, 256, 3, 2, 1, True, 1)]
    for head, cpa in (('loc', 4), ('conf', 2)):                                                     # multibox :94-106
        out += [Layer(f'{head}.0', 128, 21 * cpa, 3, 1, 1, False, 0), Layer(f'{head}.1', 256, cpa, 3, 1, 1, False, 0),
                Layer(f'{head}.2', 256, cpa, 3, 1, 1, False, 0)]
    return out


LAYERS = _layers()

# ---- the 39 launches of syn_fb_forward -----------------------------------------------------------------------------------
# kind, layer index into LAYERS (None for pools / softmax), the stages whose tensors it reads ('image' for conv1), the
# tensor it writes and the channels of it the launch owns ((lo, hi) of an NHWC map; for loc / conf the head 0..2).
Stage = namedtuple('Stage', 'kind layer inputs dest owns')


def _stages() -> List[Stage]:
    t = [Stage('conv', 0, ('image',), 'c1', (0, 48)), Stage('maxpool', None, (0,), 'p1', (0, 48)),
         Stage('conv', 1, (1,), 'c2', (0, 128)), Stage('maxpool', None, (2,), 'xa', (0, 128))]
    for b in range(3):
        x, y, L0, s0 = 3 + 8 * b, ('xb', 'xa', 'xb')[b], 2 + 7 * b, 4 + 8 * b
        t += [Stage('conv', L0 + 0, (x,), y, (0, 32)), Stage('avgpool', None, (x,), 'avg', (0, 128)),
              Stage('conv', L0 + 1, (s0 + 1,), y, (32, 64)), Stage('conv', L0 + 2, (x,), 'r1', (0, 24)),
              Stage('conv', L0 + 3, (s0 + 3,), y, (64, 96)), Stage('conv', L0 + 4, (x,), 'r2', (0, 24)),
              Stage('conv', L0 + 5, (s0 + 5,), 't3', (0, 32)), Stage('conv', L0 + 6, (s0 + 6,), y, (96, 128))]
    t += [Stage('conv', 23, (27,), 'c31', (0, 128)), Stage('conv', 24, (28,), 'c32', (0, 256)),
          Stage('conv', 25, (29,), 'c41', (0, 128)), Stage('conv', 26, (30,), 'c42', (0, 256))]
    for head, first in (('loc', 27), ('conf', 30)):
        t += [Stage('conv', first + k, (src,), head, k) for k, src in enumerate((27, 29, 31))]
    t.append(Stage('softmax', None, (37,), 'conf', None))
    return t


STAGES = _stages()
BLOCK_LAST = (11, 19, 27)                       # the stage after which each inception block's output is complete
HEAD_LAST = {'loc': 34, 'conf': 37}


def conv_out(n: int, k: int, s: int, p: int) -> int:
    return (n + 2 * p - k) // s + 1


def maps(h: int, w: int) -> Dict[str, Tuple[int, int]]:
    """(rows, columns) of every feature map of an h x w image."""
    m = {'c1': (conv_out(h, 7, 4, 3), conv_out(w, 7, 4, 3))}
    m['p1'] = tuple(conv_out(n, 3, 2, 1) for n in m['c1'])
    m['c2'] = tuple(conv_out(n, 5, 2, 2) for n in m['p1'])
    m['s0'] = tuple(conv_out(n, 3, 2, 1) for n in m['c2'])
    m['s1'] = tuple(conv_out(n, 3, 2, 1) for n in m['s0'])
    m['s2'] = tuple(conv_out(n, 3, 2, 1) for n in m['s1'])
    return m


def num_priors(h: int, w: int) -> int:
    m = maps(h, w)
    return 21 * m['s0'][0] * m['s0'][1] + m['s1'][0] * m['s1'][1] + m['s2'][0] * m['s2'][1]


def head_range(stage: int, h: int, w: int) -> Tuple[int, int]:
    """Elements [e0, e1) of the flat loc / conf that head stage ``stage`` writes."""
    st = STAGES[stage]
    m = maps(h, w)
    per = [21, 1, 1]
    n = [m[s][0] * m[s][1] * per[i] for i, s in enumerate(('s0', 's1', 's2'))]
    cpa = 4 if st.dest == 'loc' else 2
    k = st.owns
    return sum(n[:k]) * cpa, sum(n[:k + 1]) * cpa


def owned(stage: int, t: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """The part of stage ``stage``'s destination tensor ``t`` that the launch writes."""
    st = STAGES[stage]
    if st.dest in ('loc', 'conf'):
        if st.kind == 'softmax':
            return t
        e0, e1 = head_range(stage, h, w)
        return t[e0:e1]
    return t[..., st.owns[0]:st.owns[1]]


# ---- float64 stages ------------------------------------------------------------------------------------------------------

def fold(sd, index: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Layer ``index`` with its BatchNorm folded in float64: (W (cout, k*k*cin) in the kernel's (ky, kx, c) order, bias)."""
    L = LAYERS[index]
    sd = strip_prefix(sd, 'module.')
    if L.bn:
        w, b = fold_bn(sd, f'{L.name}.bn', sd[f'{L.name}.conv.weight'])
    else:
        w, b = sd[f'{L.name}.weight'].double(), sd[f'{L.name}.bias'].double()
    return w.permute(0, 2, 3, 1).reshape(L.cout, -1), b


def conv(sd, index: int, x: torch.Tensor) -> Pair:
    """Layer ``index`` on the NHWC map ``x`` (H, W, cin), or on the (H, W, 3) uint8 image for conv1 -> (want, S): an
    (HO, WO, cout) map (2 * cout channels with CReLU), flattened for the heads (the NHWC order is the priors' order)."""
    L = LAYERS[index]
    if x.dtype == torch.uint8:
        x = x.double() - torch.tensor(MEAN_BGR, dtype=torch.float64)
    w, b = fold(sd, index)
    y, s = gemm64.simt(gemm64.patches(x[None], L.k, L.stride, L.pad), w, b, L.act == 1)
    if L.act == 2:
        y, s = torch.cat([y.clamp_min(0.0), (-y).clamp_min(0.0)], 1), torch.cat([s, s], 1)
    if not L.bn:
        return y.reshape(-1), s.reshape(-1)
    ho, wo = conv_out(x.shape[0], L.k, L.stride, L.pad), conv_out(x.shape[1], L.k, L.stride, L.pad)
    return y.view(ho, wo, -1), s.view(ho, wo, -1)


def _nchw(x: torch.Tensor) -> torch.Tensor:
    return x.permute(2, 0, 1)[None]


def _nhwc(x: torch.Tensor) -> torch.Tensor:
    return x[0].permute(1, 2, 0).contiguous()


def maxpool(x: torch.Tensor) -> torch.Tensor:
    """F.max_pool2d(3, 2, 1) of the NHWC map, in x's dtype: exact."""
    return _nhwc(F.max_pool2d(_nchw(x), 3, 2, 1))


def avgpool(x: torch.Tensor) -> Pair:
    """F.avg_pool2d(3, 1, 1), divisor 9 everywhere: (want, S = sum |x| / 9)."""
    x = _nchw(x.double())
    return _nhwc(F.avg_pool2d(x, 3, 1, 1)), _nhwc(F.avg_pool2d(x.abs(), 3, 1, 1))


def softmax(logits: torch.Tensor) -> Pair:
    """Softmax over the (P, 2) class scores of the flat logits: (want, S = p (1 + |a - b|)), flat."""
    z = logits.double().view(-1, 2)
    p = torch.softmax(z, dim=1)
    return p.reshape(-1), (p * (1.0 + (z[:, :1] - z[:, 1:]).abs())).reshape(-1)


def stage(sd, index: int, inputs: List[torch.Tensor]):
    """Stage ``index`` on the tensors of its ``inputs`` stages (the image for conv1): (want, S) of the part it owns, or the
    exact fp32 result of a max-pool."""
    st = STAGES[index]
    if st.kind == 'conv':
        return conv(sd, st.layer, inputs[0])
    if st.kind == 'maxpool':
        return maxpool(inputs[0])
    if st.kind == 'avgpool':
        return avgpool(inputs[0])
    return softmax(inputs[0])


def forward64(sd, image: torch.Tensor) -> Tuple[Dict[int, torch.Tensor], torch.Tensor, torch.Tensor]:
    """The whole network in float64 from the uint8 image, stage by stage through the table: (every stage's destination
    tensor as the launch leaves it, loc (P, 4), conf (P, 2)).  Channels no launch has written yet read 0."""
    h, w = int(image.shape[0]), int(image.shape[1])
    bufs, outs = {}, {}
    p = num_priors(h, w)
    bufs['loc'], bufs['conf'] = torch.zeros(p * 4, dtype=torch.float64), torch.zeros(p * 2, dtype=torch.float64)
    for i, st in enumerate(STAGES):
        r = stage(sd, i, [image if s == 'image' else outs[s] for s in st.inputs])
        want = r[0] if isinstance(r, tuple) else r.double()
        if st.kind == 'softmax':
            bufs['conf'] = want.clone()
        elif st.dest in ('loc', 'conf'):
            e0, e1 = head_range(i, h, w)
            bufs[st.dest][e0:e1] = want
        elif st.kind == 'conv' and st.dest in ('xa', 'xb'):        # an inception branch: its slice of the block output
            if st.dest not in bufs or bufs[st.dest].shape[:2] != want.shape[:2]:
                bufs[st.dest] = torch.zeros(want.shape[:2] + (128,), dtype=torch.float64)
            bufs[st.dest][..., st.owns[0]:st.owns[1]] = want
        else:
            bufs[st.dest] = want
        outs[i] = bufs[st.dest].clone()
    return outs, bufs['loc'].view(-1, 4), bufs['conf'].view(-1, 2)


# ---- image sizes that put the kernels' edges under a check ----------------------------------------------------------------

GEMM_MAPS = ('c1', 'c2', 's0', 's1', 's2')       # the output maps fb_conv_kernel tiles: conv1, conv2, inception + conv3_1,
                                                 # conv3_2 + conv4_1, conv4_2
PRODUCTION = (720, 1080)
GOLDEN = ((250, 333), (120, 96))


def choose_sizes() -> List[Tuple[int, int]]:
    """(h, w) of the images the per-stage test runs; ``check_sizes`` states what they cover."""
    return [PRODUCTION, *GOLDEN,
            (1, 333), (1, 1),            # a one-row image, a one-pixel image: every map 1 x 1
            (1024, 1024),                # 64 = 8 x 8 cells on s2 (and 64 k rows on every map)
            (33, 993),                   # s0 = 2 x 32 = 64; conv1 2241 = 35 x 64 + 1
            (193, 961),                  # s1 = 4 x 16 = 64
            (771, 258),                  # conv2 833 = 13 x 64 + 1, s1 65 = 64 + 1; h mod 4 = 3, w mod 4 = 2
            (1079, 1023)]                # s2 = 9 x 8 = 72: two M tiles; w mod 4 = 3


def _rows(h: int, w: int, m: str) -> int:
    a, b = maps(h, w)[m]
    return a * b


def claims() -> Dict[str, Callable[[int, int], bool]]:
    """What the size set must cover, each as 'some size satisfies this': name -> predicate on (h, w)."""
    c = {}
    for m in GEMM_MAPS:
        c[f'{m}: last M tile 1 row'] = lambda h, w, m=m: _rows(h, w, m) % FB_BM == 1
        c[f'{m}: last M tile 64 rows'] = lambda h, w, m=m: _rows(h, w, m) % FB_BM == 0
        c[f'{m}: last M tile 2..63 rows'] = lambda h, w, m=m: _rows(h, w, m) % FB_BM > 1
        c[f'{m}: several M tiles'] = lambda h, w, m=m: _rows(h, w, m) > FB_BM
    for r in range(4):                                  # conv1 is stride 4, pad 3: where its last window ends
        c[f'h mod 4 = {r}'] = lambda h, w, r=r: h % 4 == r
        c[f'w mod 4 = {r}'] = lambda h, w, r=r: w % 4 == r
    for par, name in ((0, 'even'), (1, 'odd')):         # the first max-pool's border
        c[f'conv1 output height {name}'] = lambda h, w, par=par: maps(h, w)['c1'][0] % 2 == par
        c[f'conv1 output width {name}'] = lambda h, w, par=par: maps(h, w)['c1'][1] % 2 == par
    c['production 720 x 1080'] = lambda h, w: (h, w) == PRODUCTION
    for g in GOLDEN:
        c[f'golden {g[0]} x {g[1]}'] = lambda h, w, g=g: (h, w) == g
    c['one-row image'] = lambda h, w: h == 1 and w > 1
    c['1 x 1 image'] = lambda h, w: (h, w) == (1, 1)
    return c


def check_sizes(sizes) -> None:
    missing = [name for name, ok in claims().items() if not any(ok(h, w) for h, w in sizes)]
    assert not missing, f'the image sizes miss: {missing}'
