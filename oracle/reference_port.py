"""CPU oracle for the SynergyNet inference hot path.  TEST INFRASTRUCTURE ONLY.

This is a CPU restatement of the reference algorithm, used as the checker by ``tests/``,
``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference`` legs of
``bench.py``.  Nothing in ``synergynet_b200/`` may import it: the product path is the sm_90a
library and fails loudly without it.

Parity status: PINNED.  The reference has no tests or golden vectors of its own for this path
(SURVEY.md section 4), so the pin is live execution of the unmodified reference modules in the
build container: ``tests/golden/make_golden.py`` imports ``synergy3DMM.SynergyNet`` from a
scratch copy of /root/reference, loads the seeded synthetic state dict and stores the reference's
own outputs in ``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks this file against
those vectors.

The floating-point work of the reference runs inside PyTorch (ATen/oneDNN on CPU), which is a
third-party dependency that the reference leaves unpinned (setup.py:8-11; README.md:34 says
PyTorch 1.9); here it is torch 2.11.0.  The backbone is therefore restated with
``torch.nn.functional`` in fp32 on CPU -- the same kernels the reference's ``nn.Module`` calls
dispatch to -- and the 3DMM reconstruction with numpy fp32.

Each function cites the reference lines it follows (paths relative to /root/reference).
"""
from __future__ import annotations

from math import asin, atan2, cos, sqrt
from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-5          # nn.BatchNorm2d default, mobilenetv2_backbone.py:36-40
STD_SIZE = 120         # utils/params.py:33

# (t, c, n, s) -- mobilenetv2_backbone.py:108-117
_STAGES = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1),
           (6, 160, 3, 2), (6, 320, 1, 1))


def _bn(x, sd, key):
    return F.batch_norm(x, sd[key + '.running_mean'], sd[key + '.running_var'],
                        sd[key + '.weight'], sd[key + '.bias'], False, 0.0, BN_EPS)


def _conv_bn_relu6(x, sd, key, stride, groups, pad):
    """ConvBNReLU, mobilenetv2_backbone.py:33-42."""
    x = F.conv2d(x, sd[key + '.0.weight'], None, stride, pad, 1, groups)
    return F.relu6(_bn(x, sd, key + '.1'))


@torch.no_grad()
def mobilenetv2_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, prefix: str = 'I2P.backbone.',
                        return_features: bool = False, return_convs: bool = False):
    """MobileNetV2._forward_impl, mobilenetv2_backbone.py:173-189 -> (param62, pool1280).

    ``sd`` is a reference-schema state dict (CPU fp32), ``x`` is (B,3,120,120) fp32 NCHW.
    ``return_features`` adds the 19 ``features[i]`` outputs; ``return_convs`` adds the 52
    conv+BN(+ReLU6) activations in execution order (project convs with the skip already added),
    which is what ``syn_debug_forward_until`` exposes on the GPU side.
    """
    sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    feats, convs = [], []
    x = _conv_bn_relu6(x, sd, 'features.0', 2, 1, 1)                     # :127
    feats.append(x)
    convs.append(x)
    cin, blk = 32, 1
    for t, c, n, s in _STAGES:                                             # :129-134
        for i in range(n):
            stride = s if i == 0 else 1
            base = f'features.{blk}.conv'
            y, j = x, 0
            if t != 1:                                                     # InvertedResidual :58-60
                y = _conv_bn_relu6(y, sd, f'{base}.0', 1, 1, 0)
                convs.append(y)
                j = 1
            y = _conv_bn_relu6(y, sd, f'{base}.{j}', stride, y.shape[1], 1)   # :61-63
            convs.append(y)
            y = F.conv2d(y, sd[f'{base}.{j + 1}.weight'])                 # :65
            y = _bn(y, sd, f'{base}.{j + 2}')                              # :66
            x = x + y if (stride == 1 and cin == c) else y                 # :55,70-74
            feats.append(x)
            convs.append(x)
            cin, blk = c, blk + 1
    x = _conv_bn_relu6(x, sd, f'features.{blk}', 1, 1, 0)                  # :136
    feats.append(x)
    convs.append(x)
    pool = F.adaptive_avg_pool2d(x, 1).reshape(x.shape[0], -1)            # :179-180
    heads = [F.linear(pool, sd[f'{h}.1.weight'], sd[f'{h}.1.bias'])       # :184-186 (Dropout = id)
             for h in ('classifier_ori', 'classifier_shape', 'classifier_exp')]
    out = torch.cat(heads, 1)                                              # :188
    ret = (out, pool)
    if return_features:
        ret += (feats,)
    if return_convs:
        ret += (convs,)
    return ret


def parse_param_62(param: np.ndarray):
    """model_building.py:25-32 / benchmark.py:68-74 (views of a (B,62) array)."""
    p_ = param[:, :12].reshape(-1, 3, 4)
    p = p_[:, :, :3]
    offset = p_[:, :, -1].reshape(-1, 3, 1)
    alpha_shp = param[:, 12:52].reshape(-1, 40, 1)
    alpha_exp = param[:, 52:62].reshape(-1, 10, 1)
    return p, offset, alpha_shp, alpha_exp


def reconstruct_vertex_62(param: np.ndarray, pack: Dict[str, np.ndarray], whitening: bool = True,
                          dense: bool = False, transform: bool = True) -> np.ndarray:
    """model_building.py:106-139 in numpy fp32.  ``pack`` holds param_mean/param_std and either
    u_base/w_shp_base/w_exp_base (sparse) or u/w_shp/w_exp (dense).  Returns (B,3,N) fp32."""
    param = np.asarray(param, np.float32)
    if param.shape[1] != 62:
        raise RuntimeError('length of params mismatch')                   # :116-119
    if whitening:
        param = param * pack['param_std'][:62] + pack['param_mean'][:62]   # :117
    p, offset, a_shp, a_exp = parse_param_62(param)
    if dense:
        u, ws, we = pack['u'], pack['w_shp'], pack['w_exp']
    else:
        u, ws, we = pack['u_base'], pack['w_shp_base'], pack['w_exp_base']
    shape = u.reshape(1, -1, 1) + ws @ a_shp + we @ a_exp                  # :125 / :133
    n = shape.shape[1] // 3
    shape = shape.reshape(-1, n, 3).transpose(0, 2, 1)                     # view(-1,N,3).transpose(1,2)
    vertex = p @ shape + offset
    if transform:
        vertex[:, 1, :] = STD_SIZE + 1 - vertex[:, 1, :]                   # :129 / :137
    return vertex.astype(np.float32)


def gather_sparse_basis(pack3dmm: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """ParamsPack, utils/params.py:24-32: u = u_shp + u_exp and the keypoint gathers."""
    kp = pack3dmm['keypoints']
    u = pack3dmm['u_shp'] + pack3dmm['u_exp']
    return dict(param_mean=pack3dmm['param_mean'], param_std=pack3dmm['param_std'], u=u,
                w_shp=pack3dmm['w_shp'], w_exp=pack3dmm['w_exp'],
                u_base=u[kp].reshape(-1, 1), w_shp_base=pack3dmm['w_shp'][kp],
                w_exp_base=pack3dmm['w_exp'][kp], keypoints=kp)


# ---- per-face numpy API pieces used by get_all_outputs (utils/inference.py) -----------------

def crop_img(img: np.ndarray, roi_box) -> np.ndarray:
    """utils/inference.py:95-125: integer-rounded ROI with zero padding (bit-exact index work)."""
    h, w = img.shape[:2]
    sx, sy, ex, ey = [int(round(v)) for v in roi_box[:4]]
    dh, dw = ey - sy, ex - sx
    res = np.zeros((dh, dw) + img.shape[2:], dtype=np.uint8)
    dsx = -sx if sx < 0 else 0
    sx = max(sx, 0)
    dex = dw - (ex - w) if ex > w else dw
    ex = min(ex, w)
    dsy = -sy if sy < 0 else 0
    sy = max(sy, 0)
    dey = dh - (ey - h) if ey > h else dh
    ey = min(ey, h)
    res[dsy:dey, dsx:dex] = img[sy:ey, sx:ex]
    return res


def rescale_to_image(vertex: np.ndarray, roi_box) -> np.ndarray:
    """utils/inference.py:127-138 (_predict_vertices after param2vert)."""
    sx, sy, ex, ey = roi_box[:4]
    scale_x = (ex - sx) / 120
    scale_y = (ey - sy) / 120
    vertex = vertex.copy()
    vertex[0, :] = vertex[0, :] * scale_x + sx
    vertex[1, :] = vertex[1, :] * scale_y + sy
    vertex[2, :] *= (scale_x + scale_y) / 2
    return vertex


def P2sRt(P: np.ndarray):
    """utils/inference.py:33-43."""
    t3d = P[:, 3]
    R1, R2 = P[0:1, :3], P[1:2, :3]
    s = (np.linalg.norm(R1) + np.linalg.norm(R2)) / 2.0
    r1 = R1 / np.linalg.norm(R1)
    r2 = R2 / np.linalg.norm(R2)
    r3 = np.cross(r1, r2)
    return s, np.concatenate((r1, r2, r3), 0), t3d


def matrix2angle_corr(R: np.ndarray):
    """utils/inference.py:45-62 (degrees)."""
    if R[2, 0] != 1 and R[2, 0] != -1:
        x = asin(R[2, 0])
        y = atan2(R[1, 2] / cos(x), R[2, 2] / cos(x))
        z = atan2(R[0, 1] / cos(x), R[0, 0] / cos(x))
    else:
        z = 0
        if R[2, 0] == -1:
            x = np.pi / 2
            y = z + atan2(R[0, 1], R[0, 2])
        else:
            x = -np.pi / 2
            y = -z + atan2(-R[0, 1], -R[0, 2])
    return [x * 180 / np.pi, y * 180 / np.pi, z * 180 / np.pi]


def predict_pose(param: np.ndarray, pack, roi_box) -> Tuple[list, np.ndarray]:
    """utils/inference.py:86-92 + :146-157: (angles[deg], t3d in image coordinates)."""
    param = param * pack['param_std'][:62] + pack['param_mean'][:62]
    Ps = param[:12].reshape(3, -1)
    _, R, t3d = P2sRt(Ps)
    angles = matrix2angle_corr(R)
    sx, sy, ex, ey = roi_box[:4]
    t3d = t3d.copy()
    t3d[0] = t3d[0] * ((ex - sx) / 120) + sx
    t3d[1] = t3d[1] * ((ey - sy) / 120) + sy
    return angles, t3d


# ---- PointNet refinement heads and the training-forward losses ---------------------------------------------

def _pn_layer(sd, x, conv, bn):
    """F.relu(bn(conv(x))) with eval-mode BatchNorm1d, as every layer of pointnet_backbone.py:32-62 / 91-102."""
    y = F.conv1d(x, sd[f'{conv}.weight'], sd[f'{conv}.bias'])
    y = F.batch_norm(y, sd[f'{bn}.running_mean'], sd[f'{bn}.running_var'], sd[f'{bn}.weight'], sd[f'{bn}.bias'],
                     False, 0.0, BN_EPS)
    return F.relu(y)


@torch.no_grad()
def mlp_for_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, avgpool: torch.Tensor, shape_code: torch.Tensor,
                    expr_code: torch.Tensor, prefix: str = 'forwardDirection.') -> torch.Tensor:
    """MLP_for.forward, backbone_nets/pointnet_backbone.py:31-64: x (B,3,N) -> point residual (B,3,N)."""
    sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    n = x.shape[2]
    out = _pn_layer(sd, x, 'conv1', 'bn1')                                  # :32
    out = _pn_layer(sd, out, 'conv2', 'bn2')                                # :33
    point_features = out                                                    # :34
    out = _pn_layer(sd, out, 'conv3', 'bn3')
    out = _pn_layer(sd, out, 'conv4', 'bn4')
    out = _pn_layer(sd, out, 'conv5', 'bn5')
    global_features = F.max_pool1d(out, n)                                  # :38
    rep = lambda t: t.unsqueeze(2).repeat(1, 1, n) if t.dim() == 2 else t.repeat(1, 1, n)   # :39,49-56
    cat = torch.cat([point_features, rep(global_features), rep(avgpool), rep(shape_code), rep(expr_code)], 1)   # :58
    out = _pn_layer(sd, cat, 'conv6', 'bn6')
    out = _pn_layer(sd, out, 'conv7', 'bn7')
    out = _pn_layer(sd, out, 'conv8', 'bn8')
    return _pn_layer(sd, out, 'conv9', 'bn9')                               # :62 (ReLU on the output too)


@torch.no_grad()
def mlp_rev_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, prefix: str = 'reverseDirection.') -> torch.Tensor:
    """MLP_rev.forward, backbone_nets/pointnet_backbone.py:90-106: x (B,3,N) -> (B,62)."""
    sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    out = x
    for i in range(1, 6):                                                   # :91-95
        out = _pn_layer(sd, out, f'conv{i}', f'bn{i}')
    g = F.max_pool1d(out, x.shape[2])                                       # :96
    heads = [_pn_layer(sd, g, f'conv6_{i}', f'bn6_{i}') for i in (1, 2, 3)]   # :99-101
    return torch.cat(heads, 1).squeeze(2)                                   # :104


def wing_loss(pred: torch.Tensor, target: torch.Tensor, omega: float = 10, epsilon: float = 2) -> torch.Tensor:
    """WingLoss.forward, loss_definition.py:15-27."""
    import math
    n_points = pred.shape[2]
    y_hat = pred.transpose(1, 2).contiguous().view(-1, 3 * n_points)
    y = target.transpose(1, 2).contiguous().view(-1, 3 * n_points)
    delta_y = (y - y_hat).abs()
    d1, d2 = delta_y[delta_y < omega], delta_y[delta_y >= omega]
    loss1 = omega * torch.log(1 + d1 / epsilon)
    C = omega - omega * math.log(1 + omega / epsilon)
    loss2 = d2 - C
    return (loss1.sum() + loss2.sum()) / (len(loss1) + len(loss2))


def param_loss(inp: torch.Tensor, target: torch.Tensor, mode: str = 'normal') -> torch.Tensor:
    """ParamLoss.forward, loss_definition.py:35-42 (one value per sample)."""
    mse = lambda a, b: (a - b) ** 2
    if mode == 'normal':
        return torch.sqrt(mse(inp[:, :12], target[:, :12]).mean(1) + mse(inp[:, 12:], target[:, 12:]).mean(1))
    return torch.sqrt(mse(inp[:, :50], target[:, 12:62]).mean(1))          # 'only_3dmm'


@torch.no_grad()
def synergy_forward(sd: Dict[str, torch.Tensor], basis: Dict[str, np.ndarray], x: torch.Tensor, target: torch.Tensor):
    """SynergyNet.forward(input, target) in eval mode, model_building.py:141-157: the five weighted losses and the
    intermediate tensors."""
    attr, avgpool = mobilenetv2_forward(sd, x)                              # :142 (I2P.forward)
    gt = target.float()
    lmk = torch.from_numpy(reconstruct_vertex_62(attr.numpy(), basis))      # :144
    lmk_gt = torch.from_numpy(reconstruct_vertex_62(gt.numpy(), basis))     # :145
    loss = {'loss_LMK_f0': 0.05 * wing_loss(lmk, lmk_gt), 'loss_Param_In': 0.02 * param_loss(attr, gt)}   # :146-147
    residual = mlp_for_forward(sd, lmk, avgpool, attr[:, 12:52], attr[:, 52:62])   # :149
    refined = lmk + 0.05 * residual                                         # :150
    loss['loss_LMK_pointNet'] = 0.05 * wing_loss(refined, lmk_gt)           # :151
    attr_s2 = mlp_rev_forward(sd, refined)                                  # :153
    loss['loss_Param_S2'] = 0.02 * param_loss(attr_s2, gt, mode='only_3dmm')        # :154
    loss['loss_Param_S1S2'] = 0.001 * param_loss(attr_s2, attr, mode='only_3dmm')   # :155
    return loss, dict(_3D_attr=attr, avgpool=avgpool, vertex_lmk=lmk, vertex_GT_lmk=lmk_gt, point_residual=residual,
                      vertex_lmk_refined=refined, _3D_attr_S2=attr_s2)


def nme_vs_reference(lmk_new: np.ndarray, lmk_ref: np.ndarray) -> np.ndarray:
    """Landmark NME of ``lmk_new`` against ``lmk_ref`` (both (B,>=2,68) in crop coordinates)
    with the bbox-sqrt-area normaliser of benchmark_aflw2000.py:127-135."""
    out = []
    for fit, gt in zip(lmk_new, lmk_ref):
        minx, maxx = gt[0].min(), gt[0].max()
        miny, maxy = gt[1].min(), gt[1].max()
        llength = sqrt(float((maxx - minx) * (maxy - miny)))
        dis = np.sqrt(((fit[:2] - gt[:2]) ** 2).sum(0)).mean()
        out.append(dis / llength)
    return np.asarray(out, np.float32)


def max_rel_err(new, ref) -> float:
    """Parity figure of merit (BASELINE.md): max|new-ref| / max|ref|."""
    new = np.asarray(new, np.float64)
    ref = np.asarray(ref, np.float64)
    return float(np.abs(new - ref).max() / max(np.abs(ref).max(), 1e-30))


# ---- ResNet-50 backbone variant (BASELINE.json configs[4]) ---------------------------------------------------------------

@torch.no_grad()
def resnet50_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, prefix: str = 'I2P.backbone.'):
    """ResNet._forward_impl with Bottleneck blocks [3,4,6,3], backbone_nets/resnet_backbone.py:120-146,227-249.
    Returns (out102 = ori|shape|exp|tex, pooled 2048-d feature).  The adapter of the H100 shim (and of the golden
    vectors) for the (param62, avgpool) contract the reference's I2P expects is out102[:, :62], pooled."""
    sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}

    def bn(t, key):
        return F.batch_norm(t, sd[key + '.running_mean'], sd[key + '.running_var'], sd[key + '.weight'], sd[key + '.bias'],
                            False, 0.0, BN_EPS)

    x = F.relu(bn(F.conv2d(x, sd['conv1.weight'], None, 2, 3), 'bn1'))                       # :229-231
    x = F.max_pool2d(x, 3, 2, 1)                                                              # :232
    for li, (blocks, stride) in enumerate(((3, 1), (4, 2), (6, 2), (3, 2)), 1):               # :234-237
        for j in range(blocks):
            pre = f'layer{li}.{j}'
            st = stride if j == 0 else 1
            out = F.relu(bn(F.conv2d(x, sd[f'{pre}.conv1.weight']), f'{pre}.bn1'))            # :126-128
            out = F.relu(bn(F.conv2d(out, sd[f'{pre}.conv2.weight'], None, st, 1), f'{pre}.bn2'))   # :130-132
            out = bn(F.conv2d(out, sd[f'{pre}.conv3.weight']), f'{pre}.bn3')                  # :134-135
            identity = x
            if j == 0:                                                                         # :137-138
                identity = bn(F.conv2d(x, sd[f'{pre}.downsample.0.weight'], None, st), f'{pre}.downsample.1')
            x = F.relu(out + identity)                                                         # :140-141
    pooled = torch.flatten(F.adaptive_avg_pool2d(x, 1), 1)                                     # :239-240
    heads = [F.linear(pooled, sd[f'{k}.weight'], sd[f'{k}.bias']) for k in ('fc_ori', 'fc_shape', 'fc_exp', 'fc_tex')]
    return torch.cat(heads, 1), pooled                                                         # :242-246
