"""The per-stage bars of every float64 oracle and the harness the GPU stage tests share.  TEST INFRASTRUCTURE.

Each stage is fed the GPU's own output of the previous stage, so errors do not accumulate and every element of every
stage is held to |got - want| <= TAU * S, S being the stage's first-order error scale (``check64.worst``).  ``Ratios``
collects the worst ratio of every stage, ``over`` picks the stages above their kind's bar and ``report`` prints them
all.  ``stage_ratios`` runs the
MobileNetV2 backbone engines against ``block64``: the unfused engines conv by conv (52 convs), the fused engine block by
block (17 blocks, conv index 3b - 1); then the pooled feature and the 62 params.
"""
from __future__ import annotations

import types
from typing import Callable, List, Tuple

import torch

from oracle import block64, gemm64
from oracle.check64 import worst
from synergynet_b200 import _lib, synthetic
from synergynet_b200.backbone import conv_plan

# The bar: |got - want| <= TAU * S at every element, per stage kind of each table: one table per oracle, and for
# block64 one per backbone engine, under the engine's name.
TAU = {
    # block64.  S is a first-order bound, and a bound carried through the three convs of a fused block is far more
    # pessimistic than the bound of one conv (it adds |W| * S of every hidden element, while real rounding errors
    # cancel), so one TAU for both would leave the fused blocks ~40x of slack.  TAU is therefore set per engine and stage
    # kind, at most 4x the worst ratio measured on an H100 80GB HBM3 (132 SMs, 700 W power limit) over the three batches
    # of tests/test_gpu_blocks.py and the rescaled checkpoint (worst in the comment):
    'simt_fp32': {'conv': 1.3e-6,        # 3.29e-07 (conv 6)
                  'pool': 8e-7,          # 2.10e-07
                  'params': 8e-8},       # 2.00e-08
    'tc_bf16x3': {'conv': 4.9e-6,        # 1.24e-06 (conv 44, rescaled checkpoint; 1.235e-06 on the original)
                  'pool': 9e-7,          # 2.38e-07
                  'params': 9e-8},       # 2.27e-08
    'tc_fused': {'block': 1.4e-7,        # 3.54e-08 (block 2)
                 'pool': 6.9e-7,         # 1.77e-07 (tail kernel)
                 'params': 8.8e-8},      # 2.22e-08
    # The single-pass engine measures 2.06e-06 (block 15) to 3.40e-05 (block 1) and 2.46e-05 at the tail: >= 14x the bar.

    # gemm64, at most 4x the worst ratio measured on an H100 80GB HBM3 (132 SMs, 700 W power limit) over the batches,
    # both checkpoints and the kernel-level cases of tests/test_gpu_gemm_layers.py (worst in the comment):
    'gemm64': {'gemm': 8e-6,        # 3.13e-06: tc_gemm_kernel, ResNet layer4.0.conv2 (K = 4608) at B = 19; PointNet 1.67e-06
               'simt': 2e-6,        # 7.18e-07: fp32 CUDA cores, ResNet stem (K = 147); PointNet conv1 9.96e-08
               'pool': 8e-7},       # 2.39e-07: fp32 average pool
    # The ratio grows with K (the fp32 accumulation over k): 1.98e-06 for K = 2360, 2.52e-06 for a 3x3 conv with K = 2304.
    # Negative control: rowmax_in / 8 measures 2.21e-01 and rowmax_in * 2^24 2.13e-04, >= 26x the bar.

    # fb64, at most 4x the worst ratio measured on an H100 80GB HBM3 (132 SMs, 400 W power limit) over the sizes of
    # fb64.choose_sizes() (worst in the comment):
    'fb64': {'conv': 1.5e-6,      # 4.37e-07: fp32 FMA on CUDA cores, conv3_2 (K = 1152) at 720 x 1080
             'avgpool': 1e-6,     # 2.57e-07: inception2's average pool at 720 x 1080
             'softmax': 4.5e-7},  # 1.25e-07: at 193 x 961
    # Negative control (conv weights rounded to bf16 before upload, 250 x 333): 1.27e-04 at its smallest (conf.1) and
    # 1.15e-03 at its largest (inception3.branch3x3_reduce), 85x and 770x the bar.

    # recon64, at most 4x the worst ratio measured on an H100 80GB HBM3 (132 SMs, 400 W power limit) over
    # tests/test_gpu_recon.py (worst in the comment):
    'recon64': {'tc': 2.5e-6,        # 8.83e-07: tensor-core path, dense, a face 1.5x beyond the fp16 clamp (face scale 2)
                'fp32': 2e-6},       # 7.18e-07: reconstruct_kernel (engine 0), dense, the same magnitude set
    # In range the tensor-core path measures 5.3e-7 (coefficients just below the clamp) and 2.5e-7 for random faces.
    # Negative control (tests/test_recon_oracle.py, numpy emulation): one of the three passes dropped measures >= 3.7e-5,
    # coefficients clamped at 60000 instead of face-scaled 0.998: >= 15x the bar.
}
# post64 (the kernels either side of the path: pose decode, box decode, losses).  'pose_seq' holds the kernel's angles
# to the double-precision angles of the fp32 R it claims to compute (S in double ulps: a few ulps of libm); the rest hold
# fp32 results to float64 (S without the unit round-off 2^-24 = 6.0e-8, which TAU carries).  At most 4x the worst ratio
# measured on an H100 80GB HBM3 (132 SMs, 700 W power limit) over tests/test_gpu_post_oracle.py (worst in the comment):
TAU['post64'] = {'pose_seq': 6.8e-16,   # 1.70e-16: the device's double asin / cos / atan2 against the host's
                 'pose': 1.6e-7,        # 4.09e-08: the yaw sweep through the lock (the host emulation measures the same)
                 't3d': 2.2e-7,         # 5.62e-08: t * k + s with the crop box
                 'decode': 1.2e-7,      # 3.10e-08: expf (torch's CPU decode measures 2.62e-08)
                 'wing': 1.6e-7,        # 7.45e-09; the reference's own fp32 sums (torch, CPU) measure 3.8e-08
                 'param_loss': 5.8e-8}  # 1.45e-08
# Negative controls (tests/test_post_oracle.py): an FMA-contracted norm measures 2.8e-06 on 'pose_seq' (4e9 x the bar),
# the float32-trigonometry pose and a decode whose exp is 64 ulps off fail 'pose' / 'decode'.
# mbv1_64.  'gemm' and 'pool' are those of gemm64; 'dw' holds the fp32 CUDA-core stages (stem, K = 27, and the depthwise
# convs, K = 9), at most 4x the worst ratio measured on an H100 80GB HBM3 (132 SMs, 700 W power limit) over the five
# widths, the batches and both checkpoints of tests/test_gpu_mbv1.py (worst in the comment):
TAU['mbv1_64'] = {'gemm': TAU['gemm64']['gemm'],     # here: 1.96e-06 (mobilenet_2 dw6 conv_sep)
                  'pool': TAU['gemm64']['pool'],     # here: 2.25e-07
                  'dw': 1.4e-6}        # 3.56e-07: the stem of mobilenet_1 at B = 33; the depthwise convs alone 2.25e-07
# Negative controls (test_negative_controls_fail_the_bar): bf16 conv_sep weights measure 6.92e-04 (86x the gemm bar),
# rowmax_in / 8 8.93e-02 (11161x).

# The rescaled checkpoints of each oracle's tests: hidden-channel (for recon64, coefficient) scales 2^lo .. 2^hi.
WIDE = {'block64': dict(seed=7, lo=-6, hi=4),       # channel factors 2^-6 .. 2^4 on every block stream
        'gemm64': dict(seed=11, lo=-6, hi=4),
        'mbv1_64': dict(seed=11, lo=-6, hi=4),
        'recon64': dict(seed=5, lo=-8, hi=8)}
TOL = 1e-4                # params, out102 and landmarks of the rescaled checkpoints against the reference's vectors
# The PointNet heads are nine random, BatchNorm-calibrated layers in a row: they amplify a relative perturbation of their
# input ~50x (measured on the oracle: 1e-6 on the landmarks -> 4.8e-5 on point_residual), and the reference's own fp32 result
# moves by 5e-6 when the same layers run in float64.  The split-fp16 GEMMs carry 22-bit operands (8x fp32's unit
# round-off), so ~1e-4 on point_residual / the regressed parameters is the expected figure; the REFINED LANDMARKS
# (lmk + 0.05 * residual), which is what the path outputs, stay at ~1e-7.
HEAD_TOL = 3e-4
# Intermediate activations are a diagnostic, not a north_star output: the calibrated synthetic network amplifies fp32
# ordering noise to ~3e-5 per layer already (engine 0 vs the oneDNN oracle); the split-fp16 tensor-core engines measure
# 7.9e-5 at the deepest layers.  DESIGN.md section 2 quotes the bound asserted here.
LAYER_TOL = {0: 1e-4, 1: 1.5e-4, 2: 1.5e-4}

ENGINES = {'simt_fp32': _lib.ENGINE_SIMT_FP32, 'tc_bf16x3': _lib.ENGINE_TC_BF16X3, 'tc_fused': _lib.ENGINE_TC_FUSED}


class Ratios(dict):
    """{stage: (worst |got - want| / S, where it occurred, the stage's kind)}.  A stage added again keeps its largest
    ratio."""

    def add(self, kind: str, stage, got, want_s, where: Callable[[tuple], tuple] = lambda ix: ix) -> Tuple[float, tuple]:
        """Hold ``got`` to ``want_s`` = (want, S); returns this call's worst ratio and its location."""
        r, ix = worst(got, *want_s)
        loc = where(ix)
        if stage not in self or r >= self[stage][0]:
            self[stage] = (r, loc, kind)
        return r, loc


def tau(table: str, stage: str) -> float:
    """The bar of a stage named by its kind and a number (``conv6``, ``block2``, ``pool``) in TAU[table]."""
    return TAU[table][stage.rstrip('0123456789')]


def over(table: str, ratios: Ratios) -> Ratios:
    """The stages of ``ratios`` above their kind's bar in TAU[table]."""
    return Ratios({s: v for s, v in ratios.items() if v[0] > TAU[table][v[2]]})


def report(tag: str, ratios: Ratios) -> None:
    """Print the worst stage of each kind, then every stage's ratio."""
    by_kind = {}
    for s, (r, loc, kind) in ratios.items():
        if r >= by_kind.get(kind, (-1.0,))[0]:
            by_kind[kind] = (r, s, loc)
    print(f'\n[{tag}] ' + '  '.join(f'{k}: {r:.3e} at {s} {loc}' for k, (r, s, loc) in by_kind.items()))
    print('  ' + '  '.join(f'{s}={v[0]:.2e}' for s, v in ratios.items()))


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    return torch.equal(a.float().contiguous().view(torch.int32), b.float().contiguous().view(torch.int32))


def check_rowmax(out: torch.Tensor, rm, stage) -> None:
    """The row maxima a stage recorded are those of its output, bit for bit."""
    assert rm is not None and torch.equal(rm, gemm64.rowmax_bits(out)), f'rowmax of {stage}'


def face_picker(batch: int, faces: List[int], device) -> Tuple[Callable, Callable]:
    """(pick, where) for the given faces of a batch whose (rows, C) stage outputs hold the same number of rows per face:
    ``pick(t)`` takes their rows of ``t`` to the CPU, ``where(per_face)`` maps an index (row, column) of the picked rows
    to (face, row within the face, column)."""
    fidx = torch.tensor(faces, device=device)
    pick = lambda t: t.view(batch, -1, t.shape[1]).index_select(0, fidx).reshape(-1, t.shape[1]).cpu()
    where = lambda per_face: (lambda ix: (faces[ix[0] // per_face], ix[0] % per_face, ix[1]))
    return pick, where


def make_model(sd, arch: str = 'mobilenet_v2', strict: bool = True):
    """SynergyNet(args) for ``arch`` in eval mode with the checkpoint ``sd``: the whole model's state dict, or with
    strict=False the backbone's alone, whose keys are loaded under ``I2P.backbone.``."""
    from synergynet_b200 import model_building
    m = model_building.SynergyNet(types.SimpleNamespace(arch=arch, img_size=120, devices_id=[0]))
    m.load_state_dict(sd if strict else {'I2P.backbone.' + k: v for k, v in sd.items()}, strict=strict)
    return m.eval()


def seeded_crops(batch: int, seed: int) -> torch.Tensor:
    """``batch`` normalised structured crops (B, 3, 120, 120) of the given seed, on the GPU."""
    return synthetic.normalize_crops(synthetic.make_structured_crops_u8(batch, seed=seed)).cuda()


def stage_ratios(eng, fused: bool, sd, x: torch.Tensor, faces: List[int]) -> Ratios:
    """Every stage of the MobileNetV2 backbone engine ``eng`` over the given faces of batch ``x`` (on the GPU): conv by
    conv, or block by block for the fused engine."""
    fidx = torch.tensor(faces, device='cuda')
    pick = lambda t: t.index_select(0, fidx).cpu().double()
    img = pick(x)
    out = Ratios()
    if fused:
        prev = img
        for b in range(1, 18):
            got = pick(eng.debug_forward_until(x, 3 * b - 1))
            out.add('block', f'block{b}', got, block64.block(sd, b, prev))
            prev = got
        pool_want = block64.tail(sd, prev)
    else:
        got = {}
        for spec in conv_plan():
            got[spec.index] = pick(eng.debug_forward_until(x, spec.index))
            src = img if spec.index == 0 else got[spec.index - 1]
            skip = got[spec.index - 3] if spec.residual else None        # the block input, before its expand
            out.add('conv', f'conv{spec.index}', got[spec.index], block64.conv(sd, spec.index, src, skip))
        pool_want = block64.avgpool(got[len(got) - 1])
    params, pool = eng.forward(x, want_pool=True)
    pool = pick(pool)
    out.add('pool', 'pool', pool, pool_want)
    out.add('params', 'params', pick(params), block64.heads(sd, pool))
    assert eng.poll_error() == 0
    assert eng.poll_saturation(warn=False) == 0
    return out
