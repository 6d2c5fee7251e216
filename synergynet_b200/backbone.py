"""Parameter containers with the reference's checkpoint key schema, plus the layer plan.

The arithmetic of the hot path lives in the CUDA library (``csrc/``); the ``nn.Module`` classes
here only *hold* parameters under the same ``state_dict`` keys as the reference so that its
checkpoints load unchanged (SURVEY.md section 8(b); reference
``backbone_nets/mobilenetv2_backbone.py:33-74,104-158`` and
``backbone_nets/pointnet_backbone.py:7-29,67-88``).  None of them implements a torch forward:
there is deliberately no CPU/eager fallback for the product path (``GhostNetParams.forward`` and the PointNet heads'
forward call the library).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List

import torch
from torch import nn

# (expand ratio t, out channels c, repeats n, first stride s) -- mobilenetv2_backbone.py:108-117
MBV2_STAGES = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2),
               (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1))
STEM_CH, LAST_CH = 32, 1280
HEAD_DIMS = (('classifier_ori', 12), ('classifier_shape', 40), ('classifier_exp', 10))
IMG = 120


@dataclass(frozen=True)
class ConvSpec:
    """One conv+BN(+ReLU6) of the backbone, in execution order."""
    index: int          # 0..51, the order the C-ABI expects (include/synergy_b200.h)
    conv_key: str       # state_dict prefix of the Conv2d ("...weight")
    bn_key: str         # state_dict prefix of the BatchNorm2d
    kind: str           # 'stem' | 'expand' | 'dw' | 'project' | 'last'
    block: int          # features index (0..18)
    cin: int
    cout: int
    ksize: int
    stride: int
    groups: int
    relu6: bool
    h_in: int
    h_out: int
    residual: bool = False   # project conv of a block with a skip connection


def _out_size(h: int, stride: int) -> int:
    return (h + 2 - 3) // stride + 1        # 3x3, padding 1


def conv_plan(prefix: str = 'features') -> List[ConvSpec]:
    """The 52 convolutions of MobileNetV2 @120x120 (SURVEY.md section 8(a) shape table)."""
    plan: List[ConvSpec] = []

    def add(**kw):
        plan.append(ConvSpec(index=len(plan), **kw))

    h = IMG
    ho = _out_size(h, 2)
    add(conv_key=f'{prefix}.0.0', bn_key=f'{prefix}.0.1', kind='stem', block=0, cin=3,
        cout=STEM_CH, ksize=3, stride=2, groups=1, relu6=True, h_in=h, h_out=ho)
    h, cin, blk = ho, STEM_CH, 1
    for t, c, n, s in MBV2_STAGES:
        for i in range(n):
            stride = s if i == 0 else 1
            hid = cin * t
            base = f'{prefix}.{blk}.conv'
            j = 0
            if t != 1:
                add(conv_key=f'{base}.0.0', bn_key=f'{base}.0.1', kind='expand', block=blk,
                    cin=cin, cout=hid, ksize=1, stride=1, groups=1, relu6=True, h_in=h, h_out=h)
                j = 1
            ho = _out_size(h, stride)
            add(conv_key=f'{base}.{j}.0', bn_key=f'{base}.{j}.1', kind='dw', block=blk, cin=hid,
                cout=hid, ksize=3, stride=stride, groups=hid, relu6=True, h_in=h, h_out=ho)
            add(conv_key=f'{base}.{j + 1}', bn_key=f'{base}.{j + 2}', kind='project', block=blk,
                cin=hid, cout=c, ksize=1, stride=1, groups=1, relu6=False, h_in=ho, h_out=ho,
                residual=(stride == 1 and cin == c))
            h, cin, blk = ho, c, blk + 1
    add(conv_key=f'{prefix}.{blk}.0', bn_key=f'{prefix}.{blk}.1', kind='last', block=blk, cin=cin,
        cout=LAST_CH, ksize=1, stride=1, groups=1, relu6=True, h_in=h, h_out=h)
    return plan


def _conv_bn_act(cin, cout, k, stride, groups):
    return nn.Sequential(nn.Conv2d(cin, cout, k, stride, (k - 1) // 2, groups=groups, bias=False),
                         nn.BatchNorm2d(cout), nn.ReLU6(inplace=True))


class _MBConvParams(nn.Module):
    """Holds ``conv.*`` of one inverted-residual block (keys as mobilenetv2_backbone.py:58-68)."""

    def __init__(self, cin, cout, stride, t):
        super().__init__()
        hid = cin * t
        mods = []
        if t != 1:
            mods.append(_conv_bn_act(cin, hid, 1, 1, 1))
        mods += [_conv_bn_act(hid, hid, 3, stride, hid), nn.Conv2d(hid, cout, 1, bias=False),
                 nn.BatchNorm2d(cout)]
        self.conv = nn.Sequential(*mods)


class MobileNetV2Params(nn.Module):
    """State-dict twin of the reference ``MobileNetV2`` (features + three heads)."""

    def __init__(self):
        super().__init__()
        feats = [_conv_bn_act(3, STEM_CH, 3, 2, 1)]
        cin = STEM_CH
        for t, c, n, s in MBV2_STAGES:
            for i in range(n):
                feats.append(_MBConvParams(cin, c, s if i == 0 else 1, t))
                cin = c
        feats.append(_conv_bn_act(cin, LAST_CH, 1, 1, 1))
        self.features = nn.Sequential(*feats)
        self.last_channel = LAST_CH
        self.num_ori, self.num_shape, self.num_exp = (d for _, d in HEAD_DIMS)
        for name, dim in HEAD_DIMS:
            setattr(self, name, nn.Sequential(nn.Dropout(0.2), nn.Linear(LAST_CH, dim)))
        for m in self.modules():      # same distributions as mobilenetv2_backbone.py:161-171
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out')
            elif isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, 0, 0.01)
                nn.init.zeros_(m.bias)

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError('MobileNetV2Params is a parameter container; the forward pass runs in '
                           'the sm_90a library via synergynet_b200.engine.Engine')


def mobilenet_v2(pretrained: bool = False, **_):
    return MobileNetV2Params()


class _PointMLPParams(nn.Module):
    """Parameter container in the reference's key schema; ``forward`` runs in the sm_90a library through the engine
    of the model that owns the module (``_engine_provider`` is installed by ``model_building._SynergyBase``)."""
    _NET = -1

    def __init__(self, num_pts, convs, bns):
        super().__init__()
        for name, (ci, co) in convs.items():
            setattr(self, name, nn.Conv1d(ci, co, 1))
        for name, c in bns.items():
            setattr(self, name, nn.BatchNorm1d(c))
        self.num_pts = num_pts
        object.__setattr__(self, '_engine_provider', None)

    def _engine(self, t):
        if self._engine_provider is None:
            raise RuntimeError(f'{type(self).__name__}: not attached to a SynergyNet model (its engine owns the GPU state)')
        if self.num_pts != 68:
            raise RuntimeError('the sm_90a PointNet heads are built for 68 landmarks (MLP_for(68) / MLP_rev(68))')
        return self._engine_provider(t, self._NET)


class MLP_for(_PointMLPParams):
    """pointnet_backbone.py:7-64 (forwardDirection.*, 63 keys)."""
    _NET = 0

    def __init__(self, num_pts):
        chans = [(3, 64), (64, 64), (64, 64), (64, 128), (128, 1024), (2418, 512), (512, 256),
                 (256, 128), (128, 3)]
        super().__init__(num_pts, {f'conv{i + 1}': c for i, c in enumerate(chans)},
                         {f'bn{i + 1}': c[1] for i, c in enumerate(chans)})

    def forward(self, x, other_input1=None, other_input2=None, other_input3=None):
        """point_residual (B,3,68) from landmarks x (B,3,68), avgpool (B,1280), shape code (B,40), expression code (B,10)
        (pointnet_backbone.py:31-64; eval-mode BatchNorm)."""
        import torch
        params = torch.zeros((x.shape[0], 62), device=x.device, dtype=torch.float32)
        params[:, 12:52] = other_input2
        params[:, 52:62] = other_input3
        res, _ = self._engine(x).mlp_for(x, other_input1, params)
        return res if x.is_cuda else res.to(x.device)


class MLP_rev(_PointMLPParams):
    """pointnet_backbone.py:67-106 (reverseDirection.*, 56 keys)."""
    _NET = 1

    def __init__(self, num_pts):
        chans = [(3, 64), (64, 64), (64, 64), (64, 128), (128, 1024)]
        convs = {f'conv{i + 1}': c for i, c in enumerate(chans)}
        bns = {f'bn{i + 1}': c[1] for i, c in enumerate(chans)}
        for tag, dim in (('6_1', 12), ('6_2', 40), ('6_3', 10)):
            convs[f'conv{tag}'] = (1024, dim)
            bns[f'bn{tag}'] = dim
        super().__init__(num_pts, convs, bns)

    def forward(self, x, other_input1=None, other_input2=None, other_input3=None):
        """(B,62) = [rot12 | shape40 | expr10] regressed back from landmarks x (B,3,68) (pointnet_backbone.py:90-106)."""
        out = self._engine(x).mlp_rev(x)
        return out if x.is_cuda else out.to(x.device)


# ---- ResNet backbones (reference backbone_nets/resnet_backbone.py:50-391; BASELINE.json configs[4] is resnet50) ----------

# The seven factories the reference's I2P can build (model_building.py:44-45): name -> (depth, width_per_group)
RESNET_ARCHS = {'resnet18': (18, 64), 'resnet34': (34, 64), 'resnet50': (50, 64), 'resnet101': (101, 64),
                'resnet152': (152, 64), 'wide_resnet50_2': (50, 128), 'wide_resnet101_2': (101, 128)}
RESNET_LAYERS = {18: (2, 2, 2, 2), 34: (3, 4, 6, 3), 50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}


class _BasicBlock(nn.Module):
    """Keys of ``BasicBlock`` (conv1/bn1 3x3 with the stride, conv2/bn2 3x3, downsample; :50-88)."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, width_per_group=64):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample


class _Bottleneck(nn.Module):
    """Keys of ``Bottleneck`` (conv1 1x1, conv2 3x3 with the stride, conv3 1x1, downsample; :90-136)."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, width_per_group=64):
        super().__init__()
        width = planes * width_per_group // 64                              # :104
        self.conv1 = nn.Conv2d(inplanes, width, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(width)
        self.conv2 = nn.Conv2d(width, width, 3, stride, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(width)
        self.conv3 = nn.Conv2d(width, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = downsample


class ResNetParams(nn.Module):
    """Key schema of ``resnet_backbone.ResNet`` for one of the seven factories of RESNET_ARCHS (conv1/bn1,
    layer1..4.{i}.conv{1,2[,3]}/bn{1,2[,3]}[/downsample.{0,1}], fc_tex/fc_ori/fc_shape/fc_exp); parameter container, the
    forward pass runs in the sm_90a library."""

    def __init__(self, depth: int = 50, width_per_group: int = 64):
        super().__init__()
        if depth not in RESNET_LAYERS or width_per_group not in (64, 128) or (width_per_group == 128 and depth not in (50, 101)):
            raise RuntimeError(f'no ResNet ({depth}, {width_per_group}); the sm_90a library builds '
                               + ', '.join(f'{a} {v}' for a, v in RESNET_ARCHS.items()))
        self.depth, self.width_per_group = depth, width_per_group
        block = _BasicBlock if depth < 50 else _Bottleneck
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        inplanes = 64
        for li, (planes, blocks, stride) in enumerate(zip((64, 128, 256, 512), RESNET_LAYERS[depth], (1, 2, 2, 2)), 1):
            layers = []
            for j in range(blocks):                                         # :203-225
                st = stride if j == 0 else 1
                ds = None
                if st != 1 or inplanes != planes * block.expansion:
                    ds = nn.Sequential(nn.Conv2d(inplanes, planes * block.expansion, 1, st, bias=False),
                                       nn.BatchNorm2d(planes * block.expansion))
                layers.append(block(inplanes, planes, st, ds, width_per_group))
                inplanes = planes * block.expansion
            setattr(self, f'layer{li}', nn.Sequential(*layers))
        self.feature_dim = 512 * block.expansion
        self.fc_tex = nn.Linear(self.feature_dim, 40)
        self.fc_ori = nn.Linear(self.feature_dim, 12)
        self.fc_shape = nn.Linear(self.feature_dim, 40)
        self.fc_exp = nn.Linear(self.feature_dim, 10)
        for m in self.modules():                                            # resnet_backbone.py:186-191
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(f'{type(self).__name__} is a parameter container; the forward pass runs in the sm_90a library')


class ResNet50Params(ResNetParams):
    """Key schema of ``resnet_backbone.resnet50()``."""
    feature_dim = 2048

    def __init__(self):
        super().__init__(50, 64)


def resnet_conv_keys(arch: str = 'resnet50'):
    """(conv key, bn key) of the convolutions of ``arch`` in the state-dict order of the C ABI (syn_resnet_set_conv):
    conv1, then per block conv1, conv2 (, conv3) and its downsample if it has one."""
    depth, _ = RESNET_ARCHS[arch]
    names = ('1', '2') if depth < 50 else ('1', '2', '3')
    keys = [('conv1', 'bn1')]
    for li, blocks in enumerate(RESNET_LAYERS[depth], 1):
        for j in range(blocks):
            pre = f'layer{li}.{j}'
            keys += [(f'{pre}.conv{c}', f'{pre}.bn{c}') for c in names]
            if j == 0 and (li > 1 or depth >= 50):                          # stride 2, or 64 -> 256 channels in layer1
                keys.append((f'{pre}.downsample.0', f'{pre}.downsample.1'))
    return keys


def resnet50_conv_keys():
    """(conv key, bn key) of the 53 convolutions in the execution order of the C ABI (syn_resnet_set_conv)."""
    return resnet_conv_keys('resnet50')


def resnet18(pretrained: bool = False, **_):
    return ResNetParams(18, 64)


def resnet34(pretrained: bool = False, **_):
    return ResNetParams(34, 64)


def resnet50(pretrained: bool = False, **_):
    return ResNet50Params()


def resnet101(pretrained: bool = False, **_):
    return ResNetParams(101, 64)


def resnet152(pretrained: bool = False, **_):
    return ResNetParams(152, 64)


def wide_resnet50_2(pretrained: bool = False, **_):
    return ResNetParams(50, 128)


def wide_resnet101_2(pretrained: bool = False, **_):
    return ResNetParams(101, 128)


# ---- MobileNetV1 backbones (reference backbone_nets/mobilenetv1_backbone.py:21-140, prelu=False) ---------------------------

MBV1_BLOCKS = (('dw2_1', 64, 1), ('dw2_2', 128, 2), ('dw3_1', 128, 1), ('dw3_2', 256, 2), ('dw4_1', 256, 1),
               ('dw4_2', 512, 2), ('dw5_1', 512, 1), ('dw5_2', 512, 1), ('dw5_3', 512, 1), ('dw5_4', 512, 1),
               ('dw5_5', 512, 1), ('dw5_6', 1024, 2), ('dw6', 1024, 1))      # (name, out channels at width 1, stride)
MBV1_WIDTHS = {'mobilenet_2': 2.0, 'mobilenet_1': 1.0, 'mobilenet_075': 0.75, 'mobilenet_05': 0.5, 'mobilenet_025': 0.25}


class _DepthWiseBlock(nn.Module):
    """Keys of ``DepthWiseBlock`` (conv_dw, bn_dw, conv_sep, bn_sep; :21-33)."""

    def __init__(self, inplanes, planes, stride=1):
        super().__init__()
        inplanes, planes = int(inplanes), int(planes)
        self.conv_dw = nn.Conv2d(inplanes, inplanes, 3, stride, 1, groups=inplanes, bias=False)
        self.bn_dw = nn.BatchNorm2d(inplanes)
        self.conv_sep = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn_sep = nn.BatchNorm2d(planes)


class MobileNetV1Params(nn.Module):
    """Key schema of ``mobilenetv1_backbone.MobileNet(widen)`` (conv1/bn1, dw2_1 .. dw6, fc_ori/fc_shape/fc_exp/fc_tex);
    parameter container, the forward pass runs in the sm_90a library."""

    def __init__(self, widen: float = 1.0, num_classes: int = 62, input_channel: int = 3):
        super().__init__()
        if input_channel != 3:
            raise RuntimeError('the sm_90a MobileNetV1 stem is built for 3-channel crops')
        self.widen_factor = float(widen)
        self.conv1 = nn.Conv2d(input_channel, int(32 * widen), 3, 2, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(int(32 * widen))
        cin = 32
        for name, cout, stride in MBV1_BLOCKS:
            setattr(self, name, _DepthWiseBlock(cin * widen, cout * widen, stride))
            cin = cout
        self.feature_dim = int(1024 * widen)
        self.num_ori, self.num_shape, self.num_exp, self.num_texture = 12, 40, 10, 40
        self.fc_ori = nn.Linear(self.feature_dim, 12)
        self.fc_shape = nn.Linear(self.feature_dim, 40)
        self.fc_exp = nn.Linear(self.feature_dim, 10)
        self.fc_tex = nn.Linear(self.feature_dim, 40)
        for m in self.modules():                                            # mobilenetv1_backbone.py:100-106
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, (2. / n) ** 0.5)
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()

    @property
    def widen_code(self) -> int:
        """100 x the widen factor: the width argument of the C ABI (syn_mbv1_set_widen)."""
        return int(round(self.widen_factor * 100))

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError('MobileNetV1Params is a parameter container; the forward pass runs in the sm_90a library')


def mobilenet_v1_conv_keys():
    """(conv key, bn key) of the 27 convolutions in the execution order of the C ABI (syn_mbv1_set_conv)."""
    keys = [('conv1', 'bn1')]
    for name, _, _ in MBV1_BLOCKS:
        keys += [(f'{name}.conv_dw', f'{name}.bn_dw'), (f'{name}.conv_sep', f'{name}.bn_sep')]
    return keys


def mobilenet_2(num_classes=62, input_channel=3):
    return MobileNetV1Params(2.0, num_classes, input_channel)


def mobilenet_1(num_classes=62, input_channel=3):
    return MobileNetV1Params(1.0, num_classes, input_channel)


def mobilenet_075(num_classes=62, input_channel=3):
    return MobileNetV1Params(0.75, num_classes, input_channel)


def mobilenet_05(num_classes=62, input_channel=3):
    return MobileNetV1Params(0.5, num_classes, input_channel)


def mobilenet_025(num_classes=62, input_channel=3):
    return MobileNetV1Params(0.25, num_classes, input_channel)


# ---- GhostNet backbone (reference backbone_nets/ghostnet_backbone.py, ghostnet() at width 1.0) -----------------------------

# (k, exp, c, se_ratio, s) of ghostnet() (ghostnet_backbone.py:243-266), one row per GhostBottleneck, stage by stage
GHOSTNET_CFGS = [[[3, 16, 16, 0, 1]], [[3, 48, 24, 0, 2]], [[3, 72, 24, 0, 1]], [[5, 72, 40, 0.25, 2]],
                 [[5, 120, 40, 0.25, 1]], [[3, 240, 80, 0, 2]],
                 [[3, 200, 80, 0, 1], [3, 184, 80, 0, 1], [3, 184, 80, 0, 1], [3, 480, 112, 0.25, 1],
                  [3, 672, 112, 0.25, 1]],
                 [[5, 672, 160, 0.25, 2]],
                 [[5, 960, 160, 0, 1], [5, 960, 160, 0.25, 1], [5, 960, 160, 0, 1], [5, 960, 160, 0.25, 1]]]
GHOSTNET_HEADS = ('classifier_ori', 'classifier_shape', 'classifier_exp', 'classifier_texture')


def _make_divisible(v, divisor, min_value=None):
    """The channel rounding of ghostnet_backbone.py:18-31."""
    min_value = divisor if min_value is None else min_value
    new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < 0.9 * v else new_v


def _conv_bn(cin, cout, k, stride=1, groups=1):
    return [nn.Conv2d(cin, cout, k, stride, k // 2, groups=groups, bias=False), nn.BatchNorm2d(cout)]


class _GhostModule(nn.Module):
    """Keys of ``GhostModule`` (primary_conv.0/.1, cheap_operation.0/.1; :78-100)."""

    def __init__(self, inp, oup):
        super().__init__()
        init = math.ceil(oup / 2)
        self.primary_conv = nn.Sequential(*_conv_bn(inp, init, 1))
        self.cheap_operation = nn.Sequential(*_conv_bn(init, init, 3, 1, init))


class _SqueezeExcite(nn.Module):
    """Keys of ``SqueezeExcite`` (conv_reduce, conv_expand, both with bias; :41-58)."""

    def __init__(self, chs):
        super().__init__()
        red = _make_divisible(chs * 0.25, 4)
        self.conv_reduce = nn.Conv2d(chs, red, 1, bias=True)
        self.conv_expand = nn.Conv2d(red, chs, 1, bias=True)


class _GhostBottleneck(nn.Module):
    """Keys of ``GhostBottleneck`` (ghost1, conv_dw/bn_dw, se, ghost2, shortcut; :102-166)."""

    def __init__(self, cin, mid, cout, k, stride, se_ratio):
        super().__init__()
        self.ghost1 = _GhostModule(cin, mid)
        if stride > 1:
            self.conv_dw = nn.Conv2d(mid, mid, k, stride, (k - 1) // 2, groups=mid, bias=False)
            self.bn_dw = nn.BatchNorm2d(mid)
        self.se = _SqueezeExcite(mid) if se_ratio else None
        self.ghost2 = _GhostModule(mid, cout)
        if cin == cout and stride == 1:
            self.shortcut = nn.Sequential()
        else:
            self.shortcut = nn.Sequential(*_conv_bn(cin, cin, k, stride, cin), *_conv_bn(cin, cout, 1))


class _ConvBnAct(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 1, 1, 0, bias=False)
        self.bn1 = nn.BatchNorm2d(cout)


class GhostNetParams(nn.Module):
    """Key schema of ``ghostnet_backbone.GhostNet(cfgs, num_classes, width, dropout)`` (:169-233), eval mode.  Unlike the
    other parameter containers its ``forward`` works, as the reference's standalone module does: (B,3,120,120) fp32
    normalised crops or raw uint8 crops -> the (B,102) ori | shape | exp | tex output, computed in the sm_90a library.
    Only width 1.0 is built (the other widths give GEMMs with K = 12, which the tensor-core GEMM cannot take)."""

    def __init__(self, cfgs=None, num_classes: int = 1000, width: float = 1.0, dropout: float = 0.2):
        super().__init__()
        if width != 1.0:
            raise RuntimeError(f'GhostNet width {width}: the sm_90a GhostNet is built for width 1.0 only')
        self.cfgs = GHOSTNET_CFGS if cfgs is None else cfgs
        if [list(map(list, c)) for c in self.cfgs] != GHOSTNET_CFGS:
            raise RuntimeError("the sm_90a GhostNet is built for the cfgs of ghostnet_backbone.ghostnet()")
        self.dropout = dropout
        self.conv_stem = nn.Conv2d(3, 16, 3, 2, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(16)
        stages, cin = [], 16
        for cfg in self.cfgs:
            layers = []
            for k, exp, c, se_ratio, s in cfg:
                cout, mid = _make_divisible(c, 4), _make_divisible(exp, 4)
                layers.append(_GhostBottleneck(cin, mid, cout, k, s, se_ratio))
                cin = cout
            stages.append(nn.Sequential(*layers))
        stages.append(nn.Sequential(_ConvBnAct(cin, 960)))
        self.blocks = nn.Sequential(*stages)
        self.conv_head = nn.Conv2d(960, 1280, 1, 1, 0, bias=True)
        self.num_ori, self.num_shape, self.num_exp, self.num_texture = 12, 40, 10, 40
        self.classifier_ori = nn.Linear(1280, 12)
        self.classifier_shape = nn.Linear(1280, 40)
        self.classifier_exp = nn.Linear(1280, 10)
        self.classifier_texture = nn.Linear(1280, 40)
        object.__setattr__(self, '_rt', None)

    def _compute_device(self, t: torch.Tensor) -> torch.device:
        """As I2P._compute_device: the input's GPU, else the GPU the parameters live on, else the current CUDA device."""
        if t.is_cuda:
            return t.device
        w = self.conv_stem.weight
        if w.is_cuda:
            return w.device
        if not torch.cuda.is_available():
            raise RuntimeError('synergynet_b200: no CUDA device (H100) visible; there is no CPU fallback')
        return torch.device('cuda', torch.cuda.current_device())

    def _engine(self, device: torch.device):
        """The engine of ``device`` with this module's weights, handed over again when the state dict changes."""
        from .model_building import _Runtime
        if self._rt is None:
            object.__setattr__(self, '_rt', _Runtime())
            self._rt._mbv2_stub = {k: v for k, v in mobilenet_v2().state_dict().items()
                                   if not k.endswith('num_batches_tracked')}
        rt = self._rt
        eng = rt.get(device, lambda: rt._mbv2_stub, None)      # the shared library state comes from a MobileNetV2 commit
        sd = {k: v for k, v in self.state_dict(keep_vars=True).items() if not k.endswith('num_batches_tracked')}
        sig = rt._signature(list(sd.values()))
        key = (eng.device.index, 'ghostnet')
        with rt._lock:
            if rt._pn_sig.get(key) != sig or getattr(eng, '_ghost_commit_of', None) is not rt._sig.get(eng.device.index):
                eng.load_ghostnet(sd)
                rt._pn_sig[key] = sig
                eng._ghost_commit_of = rt._sig.get(eng.device.index)
        return eng

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """GhostNet.forward (:214-233) in eval mode: (B,102).  A CPU input comes back on the CPU."""
        if self.training:
            raise RuntimeError('GhostNetParams.forward runs the eval forward (BatchNorm statistics, no dropout); '
                               'call .eval() first')
        if x.dim() != 4 or tuple(x.shape[1:]) != (3, IMG, IMG):
            raise RuntimeError(f'expected (B,3,{IMG},{IMG}) crops, got {tuple(x.shape)}')
        dev = self._compute_device(x)
        out, _ = self._engine(dev).forward_ghostnet(x.to(dev))
        return out if x.is_cuda else out.to(x.device)


def ghostnet(**kwargs):
    """ghostnet_backbone.ghostnet(**kwargs) (:236-268)."""
    return GhostNetParams(GHOSTNET_CFGS, **kwargs)


def ghostnet_conv_keys():
    """(conv key, bn key or None) of the 95 convolutions in the order of the C ABI (syn_ghost_set_conv /
    syn_ghost_set_conv_bias): the state-dict order.  A None bn key marks a conv with a bias (the SE convs, conv_head)."""
    out, cin = [('conv_stem', 'bn1')], 16
    for i, cfg in enumerate(GHOSTNET_CFGS):
        for j, (k, exp, c, se, s) in enumerate(cfg):
            p = f'blocks.{i}.{j}.'
            out += [(p + 'ghost1.primary_conv.0', p + 'ghost1.primary_conv.1'),
                    (p + 'ghost1.cheap_operation.0', p + 'ghost1.cheap_operation.1')]
            if s > 1:
                out.append((p + 'conv_dw', p + 'bn_dw'))
            if se:
                out += [(p + 'se.conv_reduce', None), (p + 'se.conv_expand', None)]
            out += [(p + 'ghost2.primary_conv.0', p + 'ghost2.primary_conv.1'),
                    (p + 'ghost2.cheap_operation.0', p + 'ghost2.cheap_operation.1')]
            if not (cin == c and s == 1):
                out += [(p + 'shortcut.0', p + 'shortcut.1'), (p + 'shortcut.2', p + 'shortcut.3')]
            cin = c
    out += [('blocks.9.0.conv', 'blocks.9.0.bn1'), ('conv_head', None)]
    return out
