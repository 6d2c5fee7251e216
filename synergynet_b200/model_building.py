"""Drop-in twin of the reference ``model_building.py`` for the inference hot path.

Same class names, constructor arguments, attributes, ``state_dict`` keys and method signatures
(reference model_building.py:25-32,35-62,65-165,169-306); the arithmetic of ``forward_test`` and
``reconstruct_vertex_62`` runs in the sm_90a library through ``Engine`` -- no torch conv/matmul is
executed on the product path and nothing falls back to the CPU.
"""
from __future__ import annotations

import threading
import types
from typing import Callable, Dict, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import backbone as mobilenetv2_backbone
from .backbone import MLP_for, MLP_rev
from .engine import Engine
from .inference import (INTER_LANCZOS4, INTER_LINEAR, ImagePack, crop_resize_device, crop_resize_frames_device, crop_resize_images_device,
                        chunk_ranges, draw_lines_device, pack_images, plan_axis, roi_affine, split_by_counts, square_roi,
                        stack_frames_device)
from .params import ParamsPack, get_param_pack, set_param_pack  # noqa: F401  (re-exported)

_LOSS_KEYS = ('loss_LMK_f0', 'loss_LMK_pointNet', 'loss_Param_In', 'loss_Param_S2', 'loss_Param_S1S2')


def parse_param_62(param):
    """Views of a (B,62) tensor: rotation (B,3,3), offset (B,3,1), alpha_shp (B,40,1),
    alpha_exp (B,10,1) (reference model_building.py:25-32; index work, bit-exact)."""
    cam = param[:, :12].reshape(-1, 3, 4)
    return (cam[:, :, :3], cam[:, :, -1].reshape(-1, 3, 1),
            param[:, 12:52].reshape(-1, 40, 1), param[:, 52:62].reshape(-1, 10, 1))


class _Runtime:
    """Per-device engines for one model; rebuilt when the parameters they were packed from change
    (``load_state_dict``, in-place edits, ``.cuda()``)."""

    def __init__(self):
        self._engines: Dict[int, Engine] = {}
        self._sig: Dict[int, tuple] = {}
        self._pn_sig: Dict[tuple, tuple] = {}
        self._lock = threading.RLock()
        self.engine_kind = None      # None: the library default (fused tensor-core engine)

    @staticmethod
    def _signature(tensors) -> tuple:
        return tuple((t.data_ptr(), t._version) for t in tensors)

    def get(self, device: torch.device, backbone_sd: Callable[[], Dict[str, torch.Tensor]],
            basis: Optional[Callable[[], Dict[str, torch.Tensor]]]) -> Engine:
        if device.type != 'cuda':
            raise RuntimeError('synergynet_b200: the forward pass needs inputs on a CUDA device '
                               '(H100); there is no CPU fallback')
        idx = device.index if device.index is not None else torch.cuda.current_device()
        sd = backbone_sd()
        bs = basis() if basis is not None else {}
        sig = self._signature(list(sd.values()) + list(bs.values()))
        with self._lock:
            eng = self._engines.get(idx)
            if eng is None or self._sig.get(idx) != sig:
                if eng is None:
                    eng = Engine(idx)
                    self._engines[idx] = eng
                eng.load_backbone(sd, prefix='')
                if bs:
                    eng.load_3dmm(bs['param_mean'], bs['param_std'], bs['u_base'], bs['w_shp_base'],
                                  bs['w_exp_base'], bs.get('u'), bs.get('w_shp'), bs.get('w_exp'))
                else:   # backbone-only use: identity whitening, dummy one-point basis
                    z = torch.zeros(62)
                    eng.load_3dmm(z, z + 1, torch.zeros(3, 1), torch.zeros(3, 40), torch.zeros(3, 10))
                eng.commit()
                if self.engine_kind is not None:
                    eng.set_engine(self.engine_kind)
                self._sig[idx] = sig
                self._pn_sig.pop((idx, 0), None)          # a new commit rebuilds the library state: re-hand the heads
                self._pn_sig.pop((idx, 1), None)
        return eng

    def ensure_pointnet(self, eng: Engine, net: int, module: nn.Module) -> None:
        """Hand the PointNet head ``module`` (net 0 = MLP_for, 1 = MLP_rev) to ``eng`` when its parameters changed."""
        sd = {k: v for k, v in module.state_dict(keep_vars=True).items() if not k.endswith('num_batches_tracked')}
        sig = self._signature(list(sd.values()))
        key = (eng.device.index, net)
        with self._lock:
            if self._pn_sig.get(key) != sig:
                eng.load_pointnet(net, sd)
                self._pn_sig[key] = sig


class I2P(nn.Module):
    """Image-to-parameter module (reference model_building.py:35-62)."""

    def __init__(self, args):
        super().__init__()
        self.args = args
        if 'mobilenet_v2' in self.args.arch:
            self.backbone = getattr(mobilenetv2_backbone, args.arch)(pretrained=False)
        elif 'mobilenet' in self.args.arch:
            # the reference sends every other 'mobilenet*' arch to mobilenetv1_backbone (model_building.py:42-43).  Like
            # ResNet-50, MobileNet.forward returns ONE (B,102) tensor (mobilenetv1_backbone.py:138-140) and the reference's
            # I2P unpacks two values from it along dim 0: it raises for B != 2, and for B = 2 it silently takes face 0's
            # row as the params of both faces and face 1's as the pool.  Same adapter as resnet50: params = out[:, :62]
            # (ori|shape|exp), avgpool = the 1024w-d pooled feature.
            if self.args.arch not in mobilenetv2_backbone.MBV1_WIDTHS:
                raise RuntimeError(f"arch '{args.arch}': the MobileNetV1 backbones are "
                                   f"{', '.join(mobilenetv2_backbone.MBV1_WIDTHS)}")
            self.backbone = getattr(mobilenetv2_backbone, args.arch)()
        elif 'resnet' in self.args.arch:
            # the reference builds any 'resnet' arch with getattr(resnet_backbone, arch)(pretrained=False)
            # (model_building.py:44-45): the seven factories of RESNET_ARCHS; resnet50 is BASELINE.json configs[4].  The
            # reference's own I2P cannot run these backbones: ResNet._forward_impl returns ONE (B,102) tensor
            # (resnet_backbone.py:242-249) and I2P unpacks two (model_building.py:55,61; SURVEY.md fact 4).  Adapter used
            # here (and by the oracle / golden vectors): params = out[:, :62] (ori|shape|exp), avgpool = the pooled
            # feature (2048-d; 512-d for resnet18 / 34).
            if self.args.arch not in mobilenetv2_backbone.RESNET_ARCHS:
                raise RuntimeError(f"arch '{args.arch}': the ResNet backbones are "
                                   f"{', '.join(mobilenetv2_backbone.RESNET_ARCHS)}")
            self.backbone = getattr(mobilenetv2_backbone, args.arch)(pretrained=False)
        elif any(k in self.args.arch for k in ('ghostnet', 'resnest')):
            raise RuntimeError(f"arch '{args.arch}': mobilenet_v2 and resnet50 are built for sm_90a "
                               '(SURVEY.md section 8; the other backbones are not on the hot path)')
        else:
            raise RuntimeError("Please choose [mobilenet_v2, mobilenet_1, resnet50, or ghostnet]")
        self._is_resnet = self.args.arch in mobilenetv2_backbone.RESNET_ARCHS
        self._is_mbv1 = self.args.arch in mobilenetv2_backbone.MBV1_WIDTHS
        self._adapted = self._is_resnet or self._is_mbv1      # one (B,102) output: params = out[:, :62]
        object.__setattr__(self, '_rt', _Runtime())
        object.__setattr__(self, '_basis_provider', None)

    def _backbone_sd(self):
        return {k: v for k, v in self.backbone.state_dict(keep_vars=True).items()
                if not k.endswith('num_batches_tracked')}

    def _engine(self, device) -> Engine:
        if self._adapted:
            return self._adapted_engine(device)
        return self._rt.get(device, self._backbone_sd, self._basis_provider)

    def _adapted_engine(self, device) -> Engine:
        """Engine with the weights of the ResNet or MobileNetV1 backbone: the shared library state (error flag, 3DMM bases
        for reconstruct) comes from a commit of the MobileNetV2 path with a zero checkpoint of the right schema, then the
        backbone's layers are handed over."""
        rt = self._rt
        if not hasattr(rt, '_mbv2_stub'):
            rt._mbv2_stub = {k: v for k, v in mobilenetv2_backbone.mobilenet_v2().state_dict().items()
                             if not k.endswith('num_batches_tracked')}
        eng = rt.get(device, lambda: rt._mbv2_stub, self._basis_provider)
        sd = self._backbone_sd()
        sig = rt._signature(list(sd.values()))
        key = (eng.device.index, self.args.arch)
        with rt._lock:
            if rt._pn_sig.get(key) != sig or getattr(eng, '_adapted_commit_of', None) is not rt._sig.get(eng.device.index):
                load = eng.load_mobilenet_v1 if self._is_mbv1 else eng.load_resnet
                load(sd, self.args.arch)
                rt._pn_sig[key] = sig
                eng._adapted_commit_of = rt._sig.get(eng.device.index)
        return eng

    def _forward_adapted(self, x: torch.Tensor):
        """(out102, pool) of the ResNet / mobilenet_* backbone on ``x`` (fp32 crops or uint8 crops), which lives on the
        compute device."""
        eng = self._engine(x.device)
        return eng.forward_mobilenet_v1(x) if self._is_mbv1 else eng.forward_resnet(x)

    def _compute_device(self, t: Optional[torch.Tensor] = None) -> torch.device:
        """Where the library runs for tensor ``t``: its own GPU, else the GPU the backbone lives on, else the current
        CUDA device -- the reference wrappers are built on the CPU (synergy3DMM.py:71-77) and still usable as is."""
        if t is not None and t.is_cuda:
            return t.device
        w = next(self.backbone.parameters())
        if w.is_cuda:
            return w.device
        if not torch.cuda.is_available():
            raise RuntimeError('synergynet_b200: no CUDA device (H100) visible; there is no CPU fallback')
        return torch.device('cuda', torch.cuda.current_device())

    def forward_test(self, input):
        """Testing time forward -> (param62, avgpool1280) (model_building.py:59-62).  A CPU input is moved to the
        compute GPU and the results come back on the CPU, as the reference's CPU model would return them."""
        dev = self._compute_device(input)
        if self._adapted:
            out, pool = self._forward_adapted(input.to(dev))
            params = out[:, :62].contiguous()
        else:
            params, pool = self._engine(dev).forward(input.to(dev), want_pool=True)
        if not input.is_cuda:
            params, pool = params.to(input.device), pool.to(input.device)
        return params, pool

    def forward(self, input, target):
        """Training time forward (model_building.py:53-57): same backbone pass, GT cast."""
        params, pool = self.forward_test(input)
        return params, target.to(device=input.device, dtype=torch.float32), pool


class _SynergyBase(nn.Module):
    """Everything the two reference wrappers share: buffers, ``data_param``,
    ``reconstruct_vertex_62``, ``forward_test``, ``load_weights``, ``get_all_outputs``."""

    resize_interpolation = 'lanczos4'          # synergy3DMM.py:188; singleImage.py:77 uses linear

    def _setup(self, args, pack: ParamsPack, device: Optional[str]):
        tri = pack.tri if pack.tri is not None else np.zeros((3, 0), np.int64)
        self.triangles = torch.from_numpy(np.asarray(tri).astype(np.int64) - 1).long()
        self.I2P = I2P(args)
        self.forwardDirection = MLP_for(68)
        self.reverseDirection = MLP_rev(68)
        self.loss = {k: 0.0 for k in _LOSS_KEYS}
        for name in ('param_mean', 'param_std', 'w_shp', 'u', 'w_exp', 'u_base', 'w_shp_base', 'w_exp_base'):
            self.register_buffer(name, torch.from_numpy(np.ascontiguousarray(getattr(pack, name))).float())
        self.keypoints = torch.from_numpy(np.asarray(pack.keypoints)).long()
        self.std_size = pack.std_size
        self.face_detector = None
        if device is not None:
            self.triangles = self.triangles.to(device)
            self.to(device)
        self._refresh_data_param()
        object.__setattr__(self.I2P, '_basis_provider', self._basis)
        object.__setattr__(self.forwardDirection, '_engine_provider', self._pointnet_engine)
        object.__setattr__(self.reverseDirection, '_engine_provider', self._pointnet_engine)

    def _refresh_data_param(self):
        self.data_param = [self.param_mean, self.param_std, self.w_shp_base, self.u_base, self.w_exp_base]

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        if hasattr(self, 'param_mean'):
            self._refresh_data_param()
        return out

    def _basis(self):
        return {n: getattr(self, n) for n in ('param_mean', 'param_std', 'u_base', 'w_shp_base',
                                              'w_exp_base', 'u', 'w_shp', 'w_exp')}

    def _engine(self, device) -> Engine:
        return self.I2P._engine(device)

    def set_engine(self, kind: int) -> None:
        """0 = fp32 CUDA-core engine, 1 = wgmma split-fp16 engine (unfused), 2 = fused wgmma engine (default);
        see include/synergy_b200.h."""
        for eng in self.I2P._rt._engines.values():
            eng.set_engine(int(kind))
        self.I2P._rt.engine_kind = int(kind)

    # ---- reference API ---------------------------------------------------------------------------
    def reconstruct_vertex_62(self, param, whitening=True, dense=False, transform=True, lmk_pts=68):
        """Whitened param (B,62) -> (B,3,68) landmarks or (B,3,53215) vertices in crop image
        space (reference model_building.py:106-139)."""
        if param.shape[1] != 62:
            raise RuntimeError('length of params mismatch')
        dev = self._compute_device(param)
        out = self._engine(dev).reconstruct(param.to(dev), dense=dense, whitening=whitening, transform=transform)
        return out if param.is_cuda else out.to(param.device)

    def _compute_device(self, t: Optional[torch.Tensor] = None) -> torch.device:
        """GPU the library runs on for tensor ``t``: t's own device, else the device of the buffers, else the current
        CUDA device (the no-argument reference wrappers are constructed on the CPU, synergy3DMM.py:71-114)."""
        if t is not None and t.is_cuda:
            return t.device
        if self.param_mean.is_cuda:
            return self.param_mean.device
        if not torch.cuda.is_available():
            raise RuntimeError('synergynet_b200: no CUDA device (H100) visible; there is no CPU fallback')
        return torch.device('cuda', torch.cuda.current_device())

    def forward_test(self, input):
        """test time forward (model_building.py:159-162): whitened (B,62) parameters (on the input's device)."""
        if self.I2P._adapted:
            return self.I2P.forward_test(input)[0]
        dev = self._compute_device(input)
        out = self._engine(dev).forward(input.to(dev))
        return out if input.is_cuda else out.to(input.device)

    def forward_landmarks(self, input):
        """forward_test + reconstruct_vertex_62(dense=False) in one library call."""
        if self.I2P._adapted:
            return self.reconstruct_vertex_62(self.forward_test(input))
        dev = self._compute_device(input)
        out = self._engine(dev).forward_landmarks(input.to(dev))
        return out if input.is_cuda else out.to(input.device)

    def _pointnet_engine(self, t: torch.Tensor, net: int) -> Engine:
        """Engine of the compute device with the weights of head ``net`` (0 = forwardDirection, 1 = reverseDirection)."""
        eng = self._engine(self._compute_device(t))
        self.I2P._rt.ensure_pointnet(eng, net, self.forwardDirection if net == 0 else self.reverseDirection)
        return eng

    def forward(self, input, target):
        """The reference's training-time forward (model_building.py:141-157) in inference mode (eval BatchNorm, no
        autograd): backbone -> landmarks of prediction and ground truth -> WingLoss / ParamLoss -> MLP_for refinement
        -> MLP_rev -> the two cycle losses.  Returns the same dict of five (weighted) losses; the intermediate
        tensors are kept in ``self.last_forward`` for inspection."""
        if self.I2P._is_mbv1:
            raise RuntimeError(f'SynergyNet.forward: MLP_for.conv6 is hard-wired to a 1280-d image feature '
                               '(pointnet_backbone.py:15,58: 2418 = 64 + 1024 + 1280 + 40 + 10); the '
                               f'{self.I2P.args.arch} backbone pools {self.I2P.backbone.feature_dim} channels, so the '
                               'refinement head cannot follow it.  Use forward_test() / reconstruct_vertex_62() with it.')
        dev = self._compute_device(input)
        eng = self._engine(dev)
        _3D_attr, avgpool = self.I2P.forward_test(input.to(dev))
        if avgpool.shape[1] != 1280:
            raise RuntimeError('SynergyNet.forward: MLP_for.conv6 is hard-wired to a 1280-d image feature '
                               f'(pointnet_backbone.py:15,58: 2418 = 64 + 1024 + 1280 + 40 + 10); the {self.I2P.args.arch} '
                               f'backbone pools {avgpool.shape[1]} channels, so the refinement head cannot follow it (the '
                               'reference fails here too, SURVEY.md fact 4).  Use forward_test() / reconstruct_vertex_62() '
                               f'with {self.I2P.args.arch}.')
        _3D_attr_GT = target.to(device=dev, dtype=torch.float32)
        vertex_lmk = eng.reconstruct(_3D_attr, dense=False)
        vertex_GT_lmk = eng.reconstruct(_3D_attr_GT, dense=False)
        self.loss['loss_LMK_f0'] = 0.05 * eng.wing_loss(vertex_lmk, vertex_GT_lmk)
        self.loss['loss_Param_In'] = 0.02 * eng.param_loss(_3D_attr, _3D_attr_GT)
        eng = self._pointnet_engine(input, 0)
        point_residual, refined = eng.mlp_for(vertex_lmk, avgpool, _3D_attr)      # refined = lmk + 0.05 * residual (:150)
        self.loss['loss_LMK_pointNet'] = 0.05 * eng.wing_loss(refined, vertex_GT_lmk)
        eng = self._pointnet_engine(input, 1)
        _3D_attr_S2 = eng.mlp_rev(refined)
        self.loss['loss_Param_S2'] = 0.02 * eng.param_loss(_3D_attr_S2, _3D_attr_GT, mode='only_3dmm')
        self.loss['loss_Param_S1S2'] = 0.001 * eng.param_loss(_3D_attr_S2, _3D_attr, mode='only_3dmm')
        self.last_forward = {'_3D_attr': _3D_attr, 'avgpool': avgpool, 'vertex_lmk': vertex_lmk, 'vertex_GT_lmk': vertex_GT_lmk,
                             'point_residual': point_residual, 'vertex_lmk_refined': refined, '_3D_attr_S2': _3D_attr_S2}
        return self.loss

    def get_losses(self):
        return self.loss.keys()

    def load_weights(self, path):
        ckpt = torch.load(path, map_location=lambda storage, loc: storage)['state_dict']
        merged = self.state_dict()
        for k, v in ckpt.items():
            merged[k.replace('module.', '')] = v     # trained under DataParallel (:259-263)
        self.load_state_dict(merged, strict=False)

    def get_all_outputs(self, input, rects: Optional[Sequence[Sequence[float]]] = None):
        """3d landmarks, dense meshes and poses of every face in a BGR uint8 image
        (model_building.py:266-306 / synergy3DMM.py:167-207), batched over faces.

        ``rects`` are detector boxes ``[x0,y0,x1,y1,score]``.  The FaceBoxes detector is outside
        the hot path (SURVEY.md section 8 f3): pass ``rects`` or set ``self.face_detector``.
        """
        if rects is None:
            if self.face_detector is None:
                raise RuntimeError('no face detector configured: pass rects=[[x0,y0,x1,y1,score],...] '
                                   'or set model.face_detector to a callable(img)->rects')
            rects = self.face_detector(input)
        boxes = [square_roi(list(r)) for r in rects]
        if not boxes:
            return [], [], []
        interp = INTER_LANCZOS4 if self.resize_interpolation == 'lanczos4' else INTER_LINEAR
        # everything is batched on the GPU: one H2D of the image, crop + resize to the planar uint8 (B,3,120,120) batch
        # (OpenCV's fixed-point arithmetic, byte for byte), uint8 -> (v-127.5)/128, backbone, both reconstructions already
        # mapped to image coordinates, pose decode.  One D2H per output, no per-face arithmetic in Python.
        dev = self._compute_device()
        eng = self._engine(dev)
        image = torch.from_numpy(np.ascontiguousarray(input, dtype=np.uint8)).to(dev)    # crop_img's uint8 crops
        batch = crop_resize_device(image, boxes, (120, 120), interp)
        if self.I2P._adapted:                       # that backbone, on the uint8 crops; then the same image-space stages
            out = eng.forward_mobilenet_v1(batch)[0] if self.I2P._is_mbv1 else eng.forward_resnet(batch)[0]
            params = out[:, :62].contiguous()
        else:
            _, params = eng.forward_landmarks(batch, want_params=True)
        roi5 = torch.from_numpy(roi_affine(boxes)).to(dev)
        lmk = eng.reconstruct_image(params, roi5, dense=False).cpu().numpy()
        mesh = eng.reconstruct_image(params, roi5, dense=True).cpu().numpy()
        ang, t3d = eng.pose_decode(params, roi5)
        ang, t3d = ang.cpu().numpy(), t3d.cpu().numpy()
        eng.raise_if_error()
        return list(lmk), list(mesh), [[ang[i].tolist(), t3d[i]] for i in range(len(boxes))]

    # device memory the dense meshes of one reconstruct_image call may take in get_all_outputs_batch (638 KB per face:
    # 1682 faces); beyond it the faces are reconstructed and copied back in chunks
    dense_chunk_bytes = 1 << 30

    def get_all_outputs_batch(self, frames, rects: Optional[Sequence[Sequence[Sequence[float]]]] = None):
        """:meth:`get_all_outputs` for N equally sized BGR uint8 frames (a list, an (N,H,W,3) array, or a uint8 CUDA
        stack): a list of N ``(lmks, meshes, poses)`` triples, entry i being what ``get_all_outputs(frames[i], rects[i])``
        returns, ``([], [], [])`` for a frame without a face.

        The frames are uploaded once.  With ``rects=None`` the detector's ``detect_batch`` gets that device stack (a
        detector without one is called frame by frame).  Then one crop launch over the faces of all frames, one backbone
        call, one landmark and one dense reconstruction (the latter in chunks of faces above ``dense_chunk_bytes``), one
        pose decode.  ROIs are computed on the host in float64 exactly as the one-image call does."""
        return self._outputs(*self._frames_front(frames, rects))

    def get_all_outputs_images(self, images, rects: Optional[Sequence[Sequence[Sequence[float]]]] = None):
        """:meth:`get_all_outputs_batch` for N BGR uint8 images of any sizes (a list of host arrays or CUDA tensors): entry
        i is what ``get_all_outputs(images[i], rects[i])`` returns, ``([], [], [])`` for an image without a face.

        The images are uploaded once, packed back to back.  With ``rects=None`` the detector's ``detect_images`` gets
        that upload (a detector without one is called image by image).  Then the same single crop launch, backbone call,
        reconstructions and pose decode as :meth:`get_all_outputs_batch`."""
        return self._outputs(*self._frames_front(images, rects, ragged=True))

    def _outputs(self, eng, stack, counts, frame_index, params, roi5):
        n_faces = len(frame_index)
        if not n_faces:
            return [([], [], []) for _ in range(len(counts))]
        lmk = eng.reconstruct_image(params, roi5, dense=False).cpu().numpy()
        mesh = [eng.reconstruct_image(params[a:b], roi5[a:b], dense=True).cpu().numpy() for a, b in self._dense_chunks(eng, n_faces)]
        mesh = mesh[0] if len(mesh) == 1 else np.concatenate(mesh)
        ang, t3d = eng.pose_decode(params, roi5)
        ang, t3d = ang.cpu().numpy(), t3d.cpu().numpy()
        eng.raise_if_error()
        poses = [[ang[i].tolist(), t3d[i]] for i in range(n_faces)]
        return list(zip(split_by_counts(lmk, counts), split_by_counts(mesh, counts), split_by_counts(poses, counts)))

    def _dense_chunks(self, eng: Engine, n_faces: int) -> list:
        per_chunk = max(1, self.dense_chunk_bytes // (3 * 4 * max(eng.n_vert, 1)))
        return chunk_ranges(n_faces, per_chunk)

    def _frames_front(self, frames, rects, ragged: bool = False, rois=None):
        """The stages of :meth:`get_all_outputs_batch` up to the parameters, on the device: ``(engine, frame stack, faces
        per frame, frame of each face, whitened params (F,62), crop -> image maps (F,5))``; the last two are None when no
        frame has a face.  ``ragged``: ``frames`` is a list of images of any sizes (:meth:`get_all_outputs_images`) and
        the "stack" is their :class:`~synergynet_b200.inference.ImagePack`.  ``rois`` (one list of boxes per frame, in
        place of ``rects``): crop boxes used as given, without ``square_roi``."""
        dev = self._compute_device()
        eng = self._engine(dev)
        stack = pack_images(frames, dev) if ragged else stack_frames_device(frames, dev)
        n = len(stack) if ragged else int(stack.shape[0])
        if rois is not None:
            rects = rois
        elif rects is None:
            if self.face_detector is None:
                raise RuntimeError('no face detector configured: pass rects (one list of [x0,y0,x1,y1,score] per frame) '
                                   'or set model.face_detector')
            batched = getattr(self.face_detector, 'detect_images' if ragged else 'detect_batch', None)
            if batched is not None:
                rects = batched(stack)
            elif ragged:
                rects = [self.face_detector(stack.image(i).cpu().numpy()) for i in range(n)]
            else:
                host = stack.cpu().numpy() if isinstance(frames, torch.Tensor) else frames
                rects = [self.face_detector(host[i]) for i in range(n)]
        if len(rects) != n:
            raise ValueError(f'{len(rects)} rect lists for {n} frames')
        counts = [len(r) for r in rects]
        boxes = [list(r) if rois is not None else square_roi(list(r)) for fr in rects for r in fr]
        frame_index = [i for i, c in enumerate(counts) for _ in range(c)]
        if not boxes:
            return eng, stack, counts, frame_index, None, None
        interp = INTER_LANCZOS4 if self.resize_interpolation == 'lanczos4' else INTER_LINEAR
        if ragged:
            batch = crop_resize_images_device(stack, frame_index, boxes, (120, 120), interp)
        else:
            batch = crop_resize_frames_device(stack, frame_index, boxes, (120, 120), interp)
        if self.I2P._adapted:
            out = eng.forward_mobilenet_v1(batch)[0] if self.I2P._is_mbv1 else eng.forward_resnet(batch)[0]
            params = out[:, :62].contiguous()
        else:
            _, params = eng.forward_landmarks(batch, want_params=True)
        roi5 = torch.from_numpy(roi_affine(boxes)).to(dev)
        return eng, stack, counts, frame_index, params, roi5

    def overlay_batch(self, frames, rects: Optional[Sequence[Sequence[Sequence[float]]]] = None, alpha: float = 0.6, tex=None,
                      connectivity=None):
        """The solid-mesh overlay of every face of N equally sized BGR uint8 frames (``get_all_outputs_batch`` followed by
        ``utils/render.render`` per frame, singleImage.py's flow) in one pass: ``(blended, solid)`` (N,H,W,3) uint8 stacks,
        numpy arrays -- or CUDA tensors when ``frames`` is a CUDA stack.  Frame i's bytes are those of
        ``Sim3DR.render(frames[i], meshes_i, tri, alpha, tex=tex)`` with the dense meshes ``get_all_outputs`` returns for
        it (a frame without a face: ``solid = frame``, ``blended = cv2.addWeighted(frame, 1 - alpha, frame, alpha, 0)``).

        The dense meshes stay on the device: they are reconstructed, lit and drawn in chunks of faces above
        ``dense_chunk_bytes`` onto the same canvases (a chunk may end inside a frame), then every frame is blended once.
        ``connectivity`` (3,ntri) 0-based replaces the model's ``triangles`` as in ``render.render``."""
        front = self._frames_front(frames, rects)
        return self._overlay_stack(frames, front, alpha, self._overlay_chunks(*self._chunk_args(front), tex, connectivity))

    def overlay_images(self, images, rects: Optional[Sequence[Sequence[Sequence[float]]]] = None, alpha: float = 0.6, tex=None,
                       connectivity=None):
        """:meth:`overlay_batch` for N BGR uint8 images of any sizes: ``(blended, solid)``, two lists of N (h_i,w_i,3)
        images, numpy arrays -- or CUDA views when every input image is a CUDA tensor.  Image i's bytes are those of
        ``Sim3DR.render(images[i], meshes_i, tri, alpha, tex=tex)`` with the dense meshes ``get_all_outputs`` returns
        for it (an image without a face: ``solid = image``, ``blended = cv2.addWeighted(image, 1 - alpha, image, alpha,
        0)``).

        The images are uploaded once, packed back to back (and detected on the device by ``detect_images`` when
        ``rects`` is None).  The dense meshes are reconstructed, lit and drawn in chunks of faces above
        ``dense_chunk_bytes`` onto the packed canvases, each chunk in place on the images it touches (a chunk may end
        inside an image); then the whole pack is blended once."""
        front = self._frames_front(images, rects, ragged=True)
        return self._overlay_list(images, front, alpha, self._overlay_chunks(*self._chunk_args(front), tex, connectivity))

    @staticmethod
    def _chunk_args(front):
        eng, stack, _counts, frame_index, params, roi5 = front
        return eng, (stack.data if isinstance(stack, ImagePack) else stack).device, frame_index, params, roi5

    @staticmethod
    def _overlay_stack(frames, front, alpha, chunks):
        """Draw ``chunks`` (of :meth:`_overlay_chunks`) onto a copy of the frame stack of ``front`` and blend it."""
        from . import Sim3DR
        stack = front[1]
        solid = stack.clone()
        for r, v, col, f0, f1, chunk_counts in chunks:
            r.rasterize_frames(solid[f0:f1], v, col, chunk_counts, out=solid[f0:f1])
        blended = Sim3DR.add_weighted(stack, solid, alpha)
        if isinstance(frames, torch.Tensor) and frames.is_cuda:
            return blended, solid
        return blended.cpu().numpy(), solid.cpu().numpy()

    @staticmethod
    def _overlay_list(images, front, alpha, chunks):
        """:meth:`_overlay_stack` for the ImagePack of ``front``: two lists of images."""
        from . import Sim3DR
        pack = front[1]
        solid = ImagePack(pack.data.clone(), pack.sizes)
        for r, v, col, f0, f1, chunk_counts in chunks:
            part = solid.slice(f0, f1)
            r.rasterize_images(part, v, col, chunk_counts, out=part)
        blended = ImagePack(Sim3DR.add_weighted(pack.data, solid.data, alpha), pack.sizes)
        if all(isinstance(im, torch.Tensor) and im.is_cuda for im in images):
            return [blended.image(i) for i in range(len(pack))], [solid.image(i) for i in range(len(pack))]
        hb, hs = blended.data.cpu().numpy(), solid.data.cpu().numpy()
        split = lambda host: [host[pack.offsets[i]:pack.offsets[i + 1]].reshape(h, w, 3) for i, (h, w) in enumerate(pack.sizes)]
        return split(hb), split(hs)

    def _overlay_chunks(self, eng, device, frame_index, params, roi5, tex, connectivity, uv=None):
        """The dense meshes of the overlay, chunk by chunk of ``dense_chunk_bytes``: yields ``(renderer, vertices (F,nver,3)
        view, colours, f0, f1, meshes per frame f0..f1-1)`` for the frames f0..f1-1 the chunk draws on.  ``uv``: a
        :class:`~synergynet_b200.inference.UVMaps` -- each mesh is then its kept vertices, drawn with the layout's
        triangles and lit times its own UV texture (``tex`` and ``connectivity`` are not read).  Raises the engine's
        error flag after the last chunk."""
        from . import Sim3DR
        from .inference import RENDER_CFG
        if not frame_index:
            return
        if uv is not None:
            tri, nver = uv.layout.render_tri, uv.layout.n_keep
            keep = torch.from_numpy(uv.layout.keep).to(device)
        else:
            tri = np.asarray(connectivity).T if connectivity is not None else self.triangles.T.cpu().numpy()
            nver = eng.n_vert
        with torch.cuda.device(device):
            r = Sim3DR._renderer_for(np.ascontiguousarray(tri, dtype=np.int32), nver)
        cfg = Sim3DR._light_cfg(**RENDER_CFG)
        texture = None if tex is None or uv is not None else torch.from_numpy(np.ascontiguousarray(tex, dtype=np.float32))
        fi = np.asarray(frame_index)
        for a, b in self._dense_chunks(eng, len(frame_index)):
            v = eng.reconstruct_image(params[a:b], roi5[a:b], dense=True)
            if uv is not None:
                v = v.index_select(2, keep)                                # (F,3,n_keep): m[:, keep] of every face
                texture = uv.sample(a, b)[0]
            v = v.transpose(1, 2)
            f0, f1 = int(fi[a]), int(fi[b - 1]) + 1                   # the frames this chunk draws on, in place
            col = r.colors(v, r.normals(v), cfg, texture)
            yield r, v, col, f0, f1, np.bincount(fi[a:b] - f0, minlength=f1 - f0)
        eng.raise_if_error()

    # ---- the textured flows of artistic.py and uv_texture_realFaces.py ------------------------------------------------
    def _uv_front(self, frames, uv_maps, uv, rects, rois, ragged: bool, overlay: bool):
        """Every refusal of the ``uv_*`` methods, before any CUDA call; then :meth:`_frames_front` and the device maps."""
        from .inference import UVLayout, UVMaps, uv_maps_host
        if not isinstance(uv, UVLayout):
            raise TypeError(f'uv must be a UVLayout, got {type(uv).__name__}')
        if rects is not None and rois is not None:
            raise ValueError('give rects (detector boxes, squared as get_all_outputs squares them) or rois (crop boxes used as '
                             'given), not both')
        if rects is None and rois is None and self.face_detector is None:
            raise ValueError('give rects or rois, or set model.face_detector')
        if rois is not None:
            rois = [list(r) for r in rois]
            if any(len(fr) and not hasattr(fr[0], '__len__') for fr in rois):    # one list of boxes for every frame
                rois = [rois] * self._count_inputs(frames, ragged)
            for fr in rois:
                for r in fr:
                    if len(r) < 4 or not (r[2] > r[0] and r[3] > r[1]):
                        raise ValueError(f'ROI {list(r)} is empty: a crop box is [x0, y0, x1, y1(, score)] with x1 > x0, y1 > y0')
        n = self._count_inputs(frames, ragged)
        if uv.nver != self.u.shape[0] // 3:
            raise ValueError(f'the UV layout has {uv.nver} vertices, the model\'s dense mesh {self.u.shape[0] // 3}')
        maps = uv_maps_host(uv_maps, n, overlay)
        for i, m in enumerate(maps):
            uv.texels(m.shape[0], m.shape[1], f'UV map {i}')
        front = self._frames_front(frames, rects, ragged=ragged, rois=rois)
        frame_index = front[3]
        face_map = [0] * len(frame_index) if len(maps) == 1 else frame_index
        return front, UVMaps(uv, maps, face_map, self._chunk_args(front)[1])

    @staticmethod
    def _count_inputs(frames, ragged: bool) -> int:
        if isinstance(frames, ImagePack):
            return len(frames)
        if not ragged and hasattr(frames, 'shape') and len(frames.shape) == 4:
            return int(frames.shape[0])
        return len(frames)

    def uv_obj_batch(self, frames, uv_maps, uv, rects=None, rois=None):
        """The textured OBJ files of artistic.py / uv_texture_realFaces.py for every face of N equally sized BGR uint8 frames:
        one list of ``bytes`` per frame, one entry per face.  Face j of frame i is what
        ``write_obj_with_colors(name, m[:, keep], deletedTri, np.flip(map_i, 0)[coord_u, coord_v][keep].astype(np.float32))``
        writes, ``m`` the dense mesh ``get_all_outputs_batch`` returns for it (with ``rois``: the crop -> forward ->
        ``predict_denseVert(param, roi)`` chain of the given box).  ``uv_maps``: one (h, w, 3|4) uint8 map per frame, or one
        for all; ``uv``: a :class:`~synergynet_b200.inference.UVLayout`.  ``rects`` are detector boxes, squared as
        ``get_all_outputs`` squares them; ``rois`` are crop boxes used as given (``[[0, 0, 256, 256, 1.0]]`` is
        uv_texture_realFaces.py's), one list per frame or one list for every frame; give one or the other (or neither,
        with ``model.face_detector`` set).  artistic.py writes only the last face of an image: entry ``[-1]``.  A frame
        without a face gives ``[]`` (the script would write the previous image's mesh again; that is not reproduced).
        Scripts resize with INTER_LINEAR: set ``model.resize_interpolation = 'linear'``.  The meshes and colour tables
        never leave the device; only the text comes back."""
        front, maps = self._uv_front(frames, uv_maps, uv, rects, rois, False, False)
        return self._uv_obj(front, maps)

    def uv_obj_images(self, images, uv_maps, uv, rects=None, rois=None):
        """:meth:`uv_obj_batch` for N BGR uint8 images of any sizes."""
        front, maps = self._uv_front(images, uv_maps, uv, rects, rois, True, False)
        return self._uv_obj(front, maps)

    def _uv_obj(self, front, maps):
        from .inference import ObjTables
        eng, _stack, counts, frame_index, params, roi5 = front
        if not frame_index:
            return [[] for _ in counts]
        tables = ObjTables(maps.layout.deleted_tri, eng.n_vert, None, maps.layout.keep, len(frame_index))
        texts = []
        for a, b in self._dense_chunks(eng, len(frame_index)):
            colors = maps.sample(a, b, texture=False, colors=True)[1]
            texts += tables.encode(eng.reconstruct_image(params[a:b], roi5[a:b], dense=True), a, colors_dev=colors)
        eng.raise_if_error()
        return split_by_counts(texts, counts)

    def uv_overlay_batch(self, frames, uv_maps, uv, rects=None, rois=None, alpha: float = 0.6):
        """The textured overlay of uv_texture_realFaces.py for N equally sized BGR uint8 frames: ``(blended, solid)`` as
        :meth:`overlay_batch` returns them.  Frame i's solid image is ``overlap = frame.copy()``, then for every face j in
        rect order ``overlap = RenderPipeline(**cfg)(m_j[:, keep].T, (deletedTri - 1).T, overlap, texture=tex_j)`` with a
        fresh ``tex_j = colors_uv[keep].astype(np.float32) / 255.0`` of map i; blended is
        ``cv2.addWeighted(frame, 1 - alpha, overlap, alpha, 0)``.  With one face per frame that is
        ``utils/render.render(img, [m[:, keep]], alpha, tex=tex, connectivity=deletedTri - 1)``.  Each kept mesh is lit by
        its own extent, as the reference lights the subset it is given.  Arguments as :meth:`uv_obj_batch`; a 4-channel
        map is refused."""
        front, maps = self._uv_front(frames, uv_maps, uv, rects, rois, False, True)
        return self._overlay_stack(frames, front, alpha, self._overlay_chunks(*self._chunk_args(front), None, None, maps))

    def uv_overlay_images(self, images, uv_maps, uv, rects=None, rois=None, alpha: float = 0.6):
        """:meth:`uv_overlay_batch` for N BGR uint8 images of any sizes: two lists of images, as :meth:`overlay_images`."""
        front, maps = self._uv_front(images, uv_maps, uv, rects, rois, True, True)
        return self._overlay_list(images, front, alpha, self._overlay_chunks(*self._chunk_args(front), None, None, maps))

    def pose_overlay_batch(self, frames, rects: Optional[Sequence[Sequence[Sequence[float]]]] = None):
        """The pose image of singleImage.py:112-118 for N equally sized BGR uint8 frames in one pass: every face's axes
        drawn by ``draw_axis`` onto a copy of its frame.  Frame i's bytes are those of a loop of
        ``draw_axis(frame_i_copy, *angles, *t3d[:2], size=50, pts68=lmk)`` over the faces ``get_all_outputs_batch``
        returns for it; a frame without a face comes back unchanged.  Returns an (N,H,W,3) uint8 numpy array, or a CUDA
        tensor when ``frames`` is a CUDA stack.

        The frames are uploaded once (and detected on the device when ``rects`` is None); crops, backbone, landmarks and
        pose decode run as in ``get_all_outputs_batch``; one small copy brings back the landmarks and angles for the
        host's end-point plan (:func:`~synergynet_b200.inference.plan_axis`), one upload takes the segments, and one
        launch draws them onto a clone of the frames.  A face whose plan fails -- where the reference's draw_axis would
        raise -- raises before anything is drawn, naming the frame and the face."""
        eng, stack, counts, frame_index, params, roi5 = self._frames_front(frames, rects)
        out = self._pose_overlay(eng, stack.clone(), counts, params, roi5)
        if isinstance(frames, torch.Tensor) and frames.is_cuda:
            return out
        return out.cpu().numpy()

    def pose_overlay_images(self, images, rects: Optional[Sequence[Sequence[Sequence[float]]]] = None):
        """:meth:`pose_overlay_batch` for N BGR uint8 images of any sizes: a list of N (h_i,w_i,3) images, numpy arrays --
        or CUDA tensors when every input image is a CUDA tensor -- each with the bytes of the ``draw_axis`` loop over
        the faces ``get_all_outputs_images`` returns for it."""
        eng, pack, counts, frame_index, params, roi5 = self._frames_front(images, rects, ragged=True)
        out = self._pose_overlay(eng, ImagePack(pack.data.clone(), pack.sizes), counts, params, roi5)
        views = [out.image(i) for i in range(len(out))]
        if all(isinstance(im, torch.Tensor) and im.is_cuda for im in images):
            return views
        host = out.data.cpu().numpy()
        return [host[out.offsets[i]:out.offsets[i + 1]].reshape(h, w, 3) for i, (h, w) in enumerate(out.sizes)]

    def obj_batch(self, frames, rects: Optional[Sequence[Sequence[Sequence[float]]]] = None, keep=None, colors=None, triangles=None):
        """The OBJ file bytes of every face of N equally sized BGR uint8 frames: one list of ``bytes`` per frame, one entry
        per face.  Face j of frame i is ``write_obj(name, get_all_outputs_batch(frames)[i][1][j], tri)`` byte for byte,
        with ``tri = model.triangles + 1`` (the (3,ntri) layout of tri.mat, 1-based as meshlab reads it) unless
        ``triangles`` is given.  With ``colors`` ((n,3) for every face, or one table per face) it is
        ``write_obj_with_colors(name, mesh[:, keep], triangles, colors)`` instead -- ``keep`` alone writes
        ``write_obj`` of the kept vertices.  The dense meshes never leave the device: they are reconstructed and encoded
        in chunks of faces of ``dense_chunk_bytes``, and only the text comes back."""
        return self._obj(*self._frames_front(frames, rects), keep, colors, triangles)

    def obj_images(self, images, rects: Optional[Sequence[Sequence[Sequence[float]]]] = None, keep=None, colors=None, triangles=None):
        """:meth:`obj_batch` for N BGR uint8 images of any sizes: face j of image i is what ``write_obj`` writes for
        ``get_all_outputs_images(images)[i][1][j]``."""
        return self._obj(*self._frames_front(images, rects, ragged=True), keep, colors, triangles)

    def _obj(self, eng, stack, counts, frame_index, params, roi5, keep, colors, triangles):
        from .inference import ObjTables
        if not frame_index:
            return [[] for _ in counts]
        tri = self.triangles.cpu().numpy() + 1 if triangles is None else triangles
        tables = ObjTables(tri, eng.n_vert, colors, keep, len(frame_index))
        texts = []
        for a, b in self._dense_chunks(eng, len(frame_index)):
            texts += tables.encode(eng.reconstruct_image(params[a:b], roi5[a:b], dense=True), a)
        eng.raise_if_error()
        return split_by_counts(texts, counts)

    def _pose_overlay(self, eng, canvas, counts, params, roi5):
        """Plan every face's axes on the host and draw them onto ``canvas`` (a stack or an ImagePack), in place."""
        n_faces = sum(counts)
        if not n_faces:
            return canvas
        lmk = eng.reconstruct_image(params, roi5, dense=False)                    # (F,3,68) float32
        ang, _ = eng.pose_decode(params, roi5)                                    # (F,3) float64
        host = torch.cat([lmk.reshape(-1).view(torch.uint8), ang.reshape(-1).view(torch.uint8)]).cpu().numpy()
        eng.raise_if_error()
        nl = lmk.numel() * 4
        lmk = host[:nl].view(np.float32).reshape(tuple(lmk.shape))
        ang = host[nl:].view(np.float64).reshape(n_faces, 3)
        seg_lists, face = [], 0
        for f, c in enumerate(counts):
            segs = []
            for j in range(c):
                s, err = plan_axis(*ang[face].tolist(), lmk[face])
                if err is not None:
                    raise type(err)(f'frame {f}, face {j}: {err}') from err
                segs += s
                face += 1
            seg_lists.append(segs)
        return draw_lines_device(canvas, seg_lists)


class SynergyNet(_SynergyBase):
    """``SynergyNet(args)`` of the reference benchmark/training scripts (model_building.py:65-165):
    buffers are placed on CUDA at construction like the reference (:69,87-101)."""

    def __init__(self, args, _device: Optional[str] = 'cuda'):
        super().__init__()
        self.img_size = args.img_size
        self._setup(args, get_param_pack(), _device)


class WrapUpSynergyNet(_SynergyBase):
    """No-argument CPU-constructible wrapper (model_building.py:169-306)."""

    def __init__(self, checkpoint_fp: str = 'pretrained/best.pth.tar'):
        super().__init__()
        args = types.SimpleNamespace(arch='mobilenet_v2', checkpoint_fp=checkpoint_fp)
        self._setup(args, get_param_pack(), None)
        try:
            print('loading weights from ', args.checkpoint_fp)
            self.load_weights(args.checkpoint_fp)
        except Exception:
            pass
        self.eval()
