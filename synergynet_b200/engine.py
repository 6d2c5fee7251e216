"""Per-device handle of the sm_90a library: weight hand-over and the compute entry points.

PyTorch is used for device memory, streams and (in bench.py) ``torch.distributed`` only; all
arithmetic of the path runs in ``libsynergy_b200.so``.
"""
from __future__ import annotations

import ctypes as C
import threading
import warnings
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .backbone import (GHOSTNET_HEADS, HEAD_DIMS, MBV1_WIDTHS, RESNET_ARCHS, conv_plan, ghostnet_conv_keys,
                       mobilenet_v1_conv_keys, resnet_conv_keys)

N_PARAMS = 62


def _host_f32(t) -> torch.Tensor:
    if isinstance(t, np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(t))
    return t.detach().to(device='cpu', dtype=torch.float32).contiguous()


class StreamOrder:
    """Orders the calls of one library handle that arrive on different CUDA streams.  The handle's calls share one
    device workspace, so a call waits (on its own stream, through an event) for the device work of the previous call
    when that ran on another stream.  The caller holds the handle's lock around ``begin`` .. the C call .. ``end``.

    Under CUDA-graph capture neither records an event (it would join the graph): the caller orders replays against
    eager calls of the same handle, e.g. ``s2.wait_stream(s1)`` after a replay on ``s1``."""

    def __init__(self, device: torch.device):
        self.device = device
        self._last_stream = None
        self._last_event = None

    def begin(self) -> int:
        """The current stream of the device, ordered after the previous call; returns its handle for the C call."""
        st = torch.cuda.current_stream(self.device)
        if torch.cuda.is_current_stream_capturing():
            return st.cuda_stream
        if self._last_stream is not None and self._last_stream != st.cuda_stream:
            st.wait_event(self._last_event)
        return st.cuda_stream

    def end(self) -> None:
        """Mark the device work of the call just enqueued on the current stream."""
        if torch.cuda.is_current_stream_capturing():
            return
        st = torch.cuda.current_stream(self.device)
        if self._last_event is None:
            self._last_event = torch.cuda.Event()
        self._last_event.record(st)
        self._last_stream = st.cuda_stream

    def synchronize(self) -> None:
        """Block the host until the device work of the last call has finished."""
        if self._last_event is not None:
            self._last_event.synchronize()


class Handle:
    """One library handle bound to ``device``, created by the entry ``_CREATE`` and freed by ``_DESTROY``.  The C handle is
    not re-entrant and all its calls share one device workspace: :meth:`_call` serialises the host threads with the
    handle's lock and orders calls that arrive on different CUDA streams with a ``StreamOrder``.  A subclass sets
    ``self._lib`` before it calls this constructor."""
    _CREATE = _DESTROY = None

    def __init__(self, device: torch.device):
        self.device = device
        h = C.c_void_p()
        _lib.check(getattr(self._lib, self._CREATE)(device.index or 0, C.byref(h)))
        self._h = h
        self._lock = threading.RLock()
        self._order = StreamOrder(device)

    def close(self):
        if getattr(self, '_h', None):
            getattr(self._lib, self._DESTROY)(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def _before_stream(self) -> None:
        """Runs under the lock, on the handle's device, before :meth:`_call` takes the stream."""

    def _call(self, name: str, *args) -> None:
        """``name(handle, *args, stream)`` on the current stream of the handle's device, ordered after the handle's
        previous call; raises SynergyLibError if it fails."""
        with torch.cuda.device(self.device), self._lock:
            self._before_stream()
            _lib.check(getattr(self._lib, name)(self._h, *args, self._order.begin()))
            self._order.end()

    def _call_host(self, name: str, *args) -> None:
        """``name(handle, *args)`` for an entry that takes no stream, under the handle's lock."""
        with self._lock:
            _lib.check(getattr(self._lib, name)(self._h, *args))


def refuse_under_capture(what: str) -> None:
    """Raise SYN_ERR_STATE if the current stream is capturing a CUDA graph: for calls that run on the library's own
    streams and synchronise the host, which a graph cannot hold."""
    if torch.cuda.is_current_stream_capturing():
        raise _lib.SynergyLibError(_lib.SYN_ERR_STATE, f"{what}: runs on the library's own streams and waits on the host, "
                                                       "so it cannot be captured in a CUDA graph; call it outside the capture")


class Engine(Handle):
    """Owns one ``syn_handle_t`` bound to ``cuda:<device>``.  nn.DataParallel replicas use one engine per device, but user
    threads may share a model, hence the handle's lock."""
    _CREATE, _DESTROY = 'syn_create', 'syn_destroy'

    def __init__(self, device: int = 0):
        self._lib = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError('synergynet_b200 needs a CUDA device (H100, sm_90a); there is no '
                               'CPU fallback for the inference hot path')
        super().__init__(torch.device('cuda', int(device)))
        self.n_pts = 0
        self.n_vert = 0
        # the conv+BN backbone each family's part of the handle holds: family -> (arch, pooled feature width); the ResNet
        # part holds resnet50 until syn_resnet_select
        self._backbones: Dict[str, Tuple[str, int]] = {'resnet': ('resnet50', 2048)}
        self._keep = []
        self._host_inflight: Dict[int, tuple] = {}     # ticket -> tensors of a submitted host call (kept alive)

    # ---- weights --------------------------------------------------------------------------------
    def load_backbone(self, sd: Dict[str, torch.Tensor], prefix: str = 'I2P.backbone.') -> None:
        """Hand the 52 conv+BN pairs and the three heads of a reference-schema state dict
        (SURVEY.md section 8(b)) to the library."""
        for spec in conv_plan():
            w = _host_f32(sd[f'{prefix}{spec.conv_key}.weight'])
            bn = [_host_f32(sd[f'{prefix}{spec.bn_key}.{k}'])
                  for k in ('weight', 'bias', 'running_mean', 'running_var')]
            _lib.check(self._lib.syn_set_conv_bn(self._h, spec.index, w.data_ptr(), w.numel(),
                                                 *[t.data_ptr() for t in bn], 1e-5))
        heads = []
        for name, _ in HEAD_DIMS:
            heads += [_host_f32(sd[f'{prefix}{name}.1.weight']), _host_f32(sd[f'{prefix}{name}.1.bias'])]
        _lib.check(self._lib.syn_set_heads(self._h, *[t.data_ptr() for t in heads]))

    def load_3dmm(self, param_mean, param_std, u_base, w_shp_base, w_exp_base, u=None, w_shp=None,
                  w_exp=None) -> None:
        mean, std = _host_f32(param_mean).reshape(-1)[:62].contiguous(), _host_f32(param_std).reshape(-1)[:62].contiguous()
        _lib.check(self._lib.syn_set_whitening(self._h, mean.data_ptr(), std.data_ptr()))
        ub, wsb, web = _host_f32(u_base), _host_f32(w_shp_base), _host_f32(w_exp_base)
        self.n_pts = ub.numel() // 3
        _lib.check(self._lib.syn_set_basis_sparse(self._h, ub.data_ptr(), wsb.data_ptr(), web.data_ptr(), self.n_pts))
        if u is not None:
            ud, wsd, wed = _host_f32(u), _host_f32(w_shp), _host_f32(w_exp)
            self.n_vert = ud.numel() // 3
            _lib.check(self._lib.syn_set_basis_dense(self._h, ud.data_ptr(), wsd.data_ptr(), wed.data_ptr(), self.n_vert))

    def commit(self) -> None:
        _lib.check(self._lib.syn_commit(self._h))

    def set_engine(self, engine: int) -> None:
        _lib.check(self._lib.syn_set_engine(self._h, int(engine)))

    @property
    def engine(self) -> int:
        return self._lib.syn_get_engine(self._h)

    @property
    def launch_count(self) -> int:
        return int(self._lib.syn_launch_count(self._h))

    def set_timing(self, on: bool) -> None:
        _lib.check(self._lib.syn_set_timing(self._h, int(on)))

    def timings(self, max_entries: int = 64):
        """[(kernel label, ms)] of the last device-buffer call (needs set_timing(True) before it), at most
        ``max_entries`` launches."""
        ms = (C.c_float * max_entries)()
        names = (C.c_char_p * max_entries)()
        n = C.c_int(0)
        _lib.check(self._lib.syn_get_timings(self._h, ms, names, max_entries, C.byref(n)))
        return [(names[i].decode(), float(ms[i])) for i in range(n.value)]

    def poll_error(self) -> int:
        """Device sync + sticky in-kernel timeout flag (0 = clean)."""
        flag = C.c_int(0)
        _lib.check(self._lib.syn_poll_error(self._h, C.byref(flag)))
        return int(flag.value)

    # ---- compute --------------------------------------------------------------------------------
    def _check_x(self, x: torch.Tensor) -> torch.Tensor:
        if x.dim() != 4 or tuple(x.shape[1:]) != (3, 120, 120):
            raise RuntimeError(f'expected (B,3,120,120) input, got {tuple(x.shape)}')
        if x.device != self.device:
            raise RuntimeError(f'input on {x.device}, engine on {self.device}')
        return x.to(torch.float32).contiguous()

    def _before_stream(self) -> None:
        """Stream-ordered calls also wait for every submitted host call."""
        if not torch.cuda.is_current_stream_capturing():
            for ticket in list(self._host_inflight):     # submitted host calls run on the library's own streams and use
                _lib.check(self._lib.syn_host_wait(self._h, ticket))   # the same workspace: let them finish (tickets stay valid)

    def raise_if_error(self) -> None:
        """Cheap (no device sync) look at the sticky time-out flag of the bounded in-kernel waits; call it after a
        host-side synchronisation point (``.cpu()``, ``synchronize``) before trusting the outputs."""
        fn = getattr(self._lib, 'syn_peek_error', None)
        if fn is None:
            return
        flag = C.c_int(0)
        _lib.check(fn(self._h, C.byref(flag)))
        if flag.value:
            raise _lib.SynergyLibError(2, 'a kernel timed out in a pipeline wait; outputs are invalid '
                                          '(Engine.poll_error() reports and clears the flag)')

    def poll_saturation(self, warn: bool = True) -> int:
        """Device sync + sticky "an activation was clamped to the fp16 range" flag of the split-fp16 engines, then
        clear it.  Raised when |x| > 937.5, +-Inf or NaN reaches a clamp: the fused kernel's input (fp32 crop and
        block inputs, engines 2 and 3), the tail kernel's input (engines 2 and 3) or an expand / conv 51 input (engine
        1); and when +-Inf or NaN reaches the input of a GEMM layer (ResNets, MobileNetV1, PointNet heads) or a 3DMM
        coefficient of the dense reconstruction.  Non-zero: use ``set_engine(0)`` (fp32) for this checkpoint, or check
        the input for Inf / NaN."""
        fn = getattr(self._lib, 'syn_poll_saturation', None)
        if fn is None:
            return 0
        flag = C.c_int(0)
        _lib.check(fn(self._h, C.byref(flag)))
        if flag.value and warn:
            warnings.warn('synergynet_b200: an activation left the range of the split-fp16 tensor-core engines and was '
                          'clamped; results differ from fp32 -- use set_engine(0) for this checkpoint', RuntimeWarning)
        return int(flag.value)

    def forward(self, x: torch.Tensor, want_pool: bool = False):
        x = self._check_x(x)
        b = x.shape[0]
        params = torch.empty((b, N_PARAMS), device=self.device, dtype=torch.float32)
        pool = torch.empty((b, 1280), device=self.device, dtype=torch.float32) if want_pool else None
        self._call('syn_forward', x.data_ptr(), b, params.data_ptr(), pool.data_ptr() if want_pool else None)
        return (params, pool) if want_pool else params

    def reconstruct(self, params: torch.Tensor, dense: bool = False, whitening: bool = True,
                    transform: bool = True) -> torch.Tensor:
        if params.dim() != 2 or params.shape[1] != N_PARAMS:
            raise RuntimeError('length of params mismatch')          # model_building.py:116-119
        params = params.to(device=self.device, dtype=torch.float32).contiguous()
        b = params.shape[0]
        n = self.n_vert if dense else self.n_pts
        if n == 0:
            raise RuntimeError('dense basis not loaded' if dense else 'sparse basis not loaded')
        out = torch.empty((b, 3, n), device=self.device, dtype=torch.float32)
        self._call('syn_reconstruct', params.data_ptr(), b, int(dense), int(whitening), int(transform), out.data_ptr())
        return out

    def reconstruct_image(self, params: torch.Tensor, roi5: torch.Tensor, dense: bool = False) -> torch.Tensor:
        """reconstruct_vertex_62 + the crop -> image affine of _predict_vertices (utils/inference.py:127-138) in one
        kernel: (B,3,N) vertices in the coordinates of the original image.  ``roi5`` (B,5) fp32 = kx, sx, ky, sy, kz
        (``inference.roi_affine``)."""
        params, roi5 = self._dev_f32(params), self._dev_f32(roi5)
        b = params.shape[0]
        if params.dim() != 2 or params.shape[1] != N_PARAMS:
            raise RuntimeError('length of params mismatch')
        if tuple(roi5.shape) != (b, 5):
            raise RuntimeError(f'roi5 must be (B,5), got {tuple(roi5.shape)}')
        n = self.n_vert if dense else self.n_pts
        if n == 0:
            raise RuntimeError('dense basis not loaded' if dense else 'sparse basis not loaded')
        out = torch.empty((b, 3, n), device=self.device, dtype=torch.float32)
        self._call('syn_reconstruct_image', params.data_ptr(), b, int(dense), roi5.data_ptr(), out.data_ptr())
        return out

    def pose_decode(self, params: torch.Tensor, roi5: Optional[torch.Tensor] = None):
        """Batched parse_pose + predict_pose (utils/inference.py:33-62,86-92,146-157): (angles (B,3) float64 degrees,
        t3d (B,3) float32 -- in image coordinates when ``roi5`` is given)."""
        params = self._dev_f32(params)
        b = params.shape[0]
        if roi5 is not None:
            roi5 = self._dev_f32(roi5)
            if tuple(roi5.shape) != (b, 5):
                raise RuntimeError(f'roi5 must be (B,5), got {tuple(roi5.shape)}')
        ang = torch.empty((b, 3), device=self.device, dtype=torch.float64)
        t3d = torch.empty((b, 3), device=self.device, dtype=torch.float32)
        self._call('syn_pose_decode', params.data_ptr(), b, roi5.data_ptr() if roi5 is not None else None, ang.data_ptr(),
                   t3d.data_ptr())
        return ang, t3d

    def set_center_crop(self, margin: int) -> None:
        """CenterCrop(margin, mode='test') of the reference loader for the uint8 entry points (0 = off)."""
        _lib.check(self._lib.syn_set_center_crop(self._h, int(margin)))

    def forward_landmarks(self, x: torch.Tensor, want_params: bool = False):
        """x: fp32 normalised crops, or raw uint8 crops (normalised on the device)."""
        if x.dtype == torch.uint8:
            return self._forward_landmarks_u8(x, want_params)
        x = self._check_x(x)
        b = x.shape[0]
        lmk = torch.empty((b, 3, self.n_pts), device=self.device, dtype=torch.float32)
        params = torch.empty((b, N_PARAMS), device=self.device, dtype=torch.float32) if want_params else None
        self._call('syn_forward_landmarks', x.data_ptr(), b, params.data_ptr() if want_params else None, lmk.data_ptr())
        return (lmk, params) if want_params else lmk

    def _forward_landmarks_u8(self, x: torch.Tensor, want_params: bool):
        if x.dim() != 4 or tuple(x.shape[1:]) != (3, 120, 120) or x.device != self.device:
            raise RuntimeError(f'expected uint8 (B,3,120,120) on {self.device}, got {tuple(x.shape)} on {x.device}')
        x = x.contiguous()
        b = x.shape[0]
        lmk = torch.empty((b, 3, self.n_pts), device=self.device, dtype=torch.float32)
        params = torch.empty((b, N_PARAMS), device=self.device, dtype=torch.float32) if want_params else None
        self._call('syn_forward_landmarks_u8', x.data_ptr(), b, params.data_ptr() if want_params else None, lmk.data_ptr())
        return (lmk, params) if want_params else lmk

    def forward_landmarks_host(self, x_host: torch.Tensor, lmk_host: Optional[torch.Tensor] = None,
                               params_host: Optional[torch.Tensor] = None) -> torch.Tensor:
        """End-to-end call on HOST tensors (pinned recommended): H2D, forward, landmarks, D2H.  Synchronous."""
        return self.host_wait(self.forward_landmarks_host_submit(x_host, lmk_host, params_host))

    def forward_landmarks_host_submit(self, x_host: torch.Tensor, lmk_host: Optional[torch.Tensor] = None,
                                      params_host: Optional[torch.Tensor] = None) -> int:
        """Enqueue the end-to-end call and return a ticket for :meth:`host_wait`.  Up to two calls may be in flight: the
        second one's host->device copies run under the first one's kernels (a loader loop: submit batch k+1, then wait
        for batch k).  The tensors are kept alive here until their ticket has been waited for."""
        if x_host.is_cuda or x_host.dtype not in (torch.float32, torch.uint8) or not x_host.is_contiguous():
            raise RuntimeError('x_host must be a contiguous fp32 (normalised) or uint8 (raw) CPU tensor')
        if x_host.dim() != 4 or tuple(x_host.shape[1:]) != (3, 120, 120):
            raise RuntimeError(f'expected (B,3,120,120) crops, got {tuple(x_host.shape)}')
        b = x_host.shape[0]
        refuse_under_capture(f'forward_landmarks_host: batch {b}')
        if lmk_host is None:
            lmk_host = torch.empty((b, 3, self.n_pts), dtype=torch.float32)
        # the C side writes B*3*n_pts and B*62 floats through these pointers: refuse anything it could overrun
        for name, buf, need in (('lmk_host', lmk_host, b * 3 * self.n_pts), ('params_host', params_host, b * N_PARAMS)):
            if buf is None:
                continue
            if buf.is_cuda or buf.dtype != torch.float32 or not buf.is_contiguous() or buf.numel() < need:
                raise RuntimeError(f'{name} must be a contiguous CPU float32 tensor with at least {need} elements')
        ticket = C.c_int(0)
        with self._lock:
            self._order.synchronize()                # stream-ordered calls share the workspace with the host pipeline
            _lib.check(self._lib.syn_forward_landmarks_host_submit(
                self._h, x_host.data_ptr(), 1 if x_host.dtype == torch.uint8 else 0, b,
                params_host.data_ptr() if params_host is not None else None, lmk_host.data_ptr(), C.byref(ticket)))
            self._host_inflight[ticket.value] = (x_host, lmk_host, params_host)
        return ticket.value

    def host_wait(self, ticket: int) -> torch.Tensor:
        """Block until the call behind ``ticket`` has written its host outputs; returns its landmark tensor."""
        with self._lock:
            if ticket not in self._host_inflight:
                raise RuntimeError(f'unknown or already collected ticket {ticket}')
            try:
                _lib.check(self._lib.syn_host_wait(self._h, ticket))
            finally:
                _, lmk_host, _ = self._host_inflight.pop(ticket)
        return lmk_host

    # ---- PointNet refinement heads + losses (training-forward surface, model_building.py:141-157) --------------
    _FOR_LAYERS = [f'conv{i}' for i in range(1, 10)]
    _REV_LAYERS = ['conv1', 'conv2', 'conv3', 'conv4', 'conv5', 'conv6_1', 'conv6_2', 'conv6_3']

    def load_pointnet(self, net: int, sd: Dict[str, torch.Tensor]) -> None:
        """net 0: MLP_for state dict (conv1..conv9 + bn1..bn9), net 1: MLP_rev (conv1..5, conv6_1/2/3 + their BN);
        keys without prefix, as ``module.state_dict()`` returns them (pointnet_backbone.py:7-29,67-88)."""
        names = self._FOR_LAYERS if net == 0 else self._REV_LAYERS
        with self._lock:                 # held across the hand-over: another thread's layers never mix with these
            for i, cname in enumerate(names):
                bname = 'bn' + cname[4:]
                w = _host_f32(sd[f'{cname}.weight'])
                cb = _host_f32(sd[f'{cname}.bias'])
                bn = [_host_f32(sd[f'{bname}.{k}']) for k in ('weight', 'bias', 'running_mean', 'running_var')]
                self._call_host('syn_pointnet_set_layer', net, i, w.data_ptr(), w.shape[0], w.shape[1], cb.data_ptr(),
                                *[t.data_ptr() for t in bn], 1e-5)
            self._call_host('syn_pointnet_commit', net)

    def _dev_f32(self, t: torch.Tensor) -> torch.Tensor:
        return t.to(device=self.device, dtype=torch.float32).contiguous()

    def mlp_for(self, lmk: torch.Tensor, pool: torch.Tensor, params: torch.Tensor):
        """(point_residual (B,3,68), lmk + 0.05 * point_residual) -- MLP_for.forward + model_building.py:150."""
        lmk, pool, params = self._dev_f32(lmk), self._dev_f32(pool), self._dev_f32(params)
        b = lmk.shape[0]
        if tuple(lmk.shape[1:]) != (3, 68) or tuple(pool.shape) != (b, 1280) or tuple(params.shape) != (b, N_PARAMS):
            raise RuntimeError(f'mlp_for: expected (B,3,68), (B,1280), (B,62); got {tuple(lmk.shape)}, {tuple(pool.shape)}, {tuple(params.shape)}')
        res, ref = torch.empty_like(lmk), torch.empty_like(lmk)
        self._call('syn_mlp_for', lmk.data_ptr(), pool.data_ptr(), params.data_ptr(), b, res.data_ptr(), ref.data_ptr())
        return res, ref

    def mlp_rev(self, lmk: torch.Tensor) -> torch.Tensor:
        lmk = self._dev_f32(lmk)
        if lmk.dim() != 3 or tuple(lmk.shape[1:]) != (3, 68):
            raise RuntimeError(f'mlp_rev: expected (B,3,68), got {tuple(lmk.shape)}')
        out = torch.empty((lmk.shape[0], N_PARAMS), device=self.device, dtype=torch.float32)
        self._call('syn_mlp_rev', lmk.data_ptr(), lmk.shape[0], out.data_ptr())
        return out

    def wing_loss(self, pred: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """WingLoss(omega=10, epsilon=2) of two (B,3,N) tensors -> 0-d tensor (loss_definition.py:8-27)."""
        pred, target = self._dev_f32(pred), self._dev_f32(target)
        if pred.shape != target.shape or pred.dim() != 3 or pred.shape[1] != 3:
            raise RuntimeError(f'wing_loss: expected two (B,3,N) tensors, got {tuple(pred.shape)} and {tuple(target.shape)}')
        out = torch.empty((1,), device=self.device, dtype=torch.float32)
        self._call('syn_wing_loss', pred.data_ptr(), target.data_ptr(), pred.shape[0], pred.shape[2], out.data_ptr())
        return out[0]

    def param_loss(self, inp: torch.Tensor, target: torch.Tensor, mode: str = 'normal') -> torch.Tensor:
        """ParamLoss (loss_definition.py:29-42): per-sample (B,) tensor; mode 'normal' or 'only_3dmm'."""
        if mode not in ('normal', 'only_3dmm'):
            raise RuntimeError(f"param_loss: mode must be 'normal' or 'only_3dmm', got {mode!r}")
        inp, target = self._dev_f32(inp), self._dev_f32(target)
        if inp.dim() != 2 or inp.shape[1] != N_PARAMS or target.shape != inp.shape:
            raise RuntimeError('param_loss: expected two (B,62) tensors')
        out = torch.empty((inp.shape[0],), device=self.device, dtype=torch.float32)
        self._call('syn_param_loss', inp.data_ptr(), target.data_ptr(), inp.shape[0], 0 if mode == 'normal' else 1,
                   out.data_ptr())
        return out

    # ---- conv+BN backbones: ResNet, MobileNetV1 and GhostNet, one (B,102) output ori | shape | exp | tex ---------------------
    def _load_convbn(self, family: str, arch: str, select, conv_keys, feat: int, sd: Dict[str, torch.Tensor],
                     prefix: str) -> None:
        """Select the plan of ``arch`` (``select``: the entry's name and its arguments after the handle), then hand over its
        conv+BN pairs in plan order and the four Linear heads concatenated in the reference's output order as (102, feat)
        weights, and commit."""
        with self._lock:                 # held across the hand-over: another thread's layers never mix with these
            self._call_host(*select)
            self._backbones[family] = (arch, feat)
            for i, (ck, bk) in enumerate(conv_keys):
                w = _host_f32(sd[f'{prefix}{ck}.weight'])
                bn = [_host_f32(sd[f'{prefix}{bk}.{k}']) for k in ('weight', 'bias', 'running_mean', 'running_var')]
                self._call_host(f'syn_{family}_set_conv', i, w.data_ptr(), w.numel(), *[t.data_ptr() for t in bn], 1e-5)
            order = ('fc_ori', 'fc_shape', 'fc_exp', 'fc_tex')
            w = torch.cat([_host_f32(sd[f'{prefix}{k}.weight']) for k in order]).contiguous()
            b = torch.cat([_host_f32(sd[f'{prefix}{k}.bias']) for k in order]).contiguous()
            if tuple(w.shape) != (102, feat):
                raise RuntimeError(f'{arch} heads: expected (102, {feat}) weights, got {tuple(w.shape)}')
            self._call_host(f'syn_{family}_set_heads', w.data_ptr(), b.data_ptr())
            self._call_host(f'syn_{family}_commit')

    def _backbone(self, family: str) -> Tuple[str, int]:
        if family not in self._backbones:
            raise RuntimeError(f'no {family} backbone loaded on this engine')
        return self._backbones[family]

    def _forward_convbn(self, family: str, x: torch.Tensor):
        """(B,3,120,120) fp32 normalised crops or raw uint8 crops -> ((B,102) out, (B,feat) pooled)."""
        if x.dtype == torch.uint8:
            if x.dim() != 4 or tuple(x.shape[1:]) != (3, 120, 120) or x.device != self.device:
                raise RuntimeError(f'expected uint8 (B,3,120,120) on {self.device}, got {tuple(x.shape)} on {x.device}')
            x = x.contiguous()
        else:
            x = self._check_x(x)
        b = x.shape[0]
        out = torch.empty((b, 102), device=self.device, dtype=torch.float32)
        pool = torch.empty((b, self._backbone(family)[1]), device=self.device, dtype=torch.float32)
        self._call(f'syn_{family}_forward', x.data_ptr(), int(x.dtype == torch.uint8), b, out.data_ptr(), pool.data_ptr())
        return out, pool

    def _debug_run(self, name: str, x: torch.Tensor, stage: int, rows: int, cols: int, rowmax: bool):
        """One syn_debug_*_until run of a conv+BN backbone on fp32 crops ``x`` into (rows, cols) and, if the stage records
        them, (rows,) row maxima."""
        out, rmax = self._debug_out(rows, cols, rowmax)
        self._call(name, x.data_ptr(), x.shape[0], stage, out.data_ptr(), rmax.data_ptr() if rowmax else None)
        return out, rmax

    # ResNet backbones (backbone_nets/resnet_backbone.py; BASELINE.json configs[4] is resnet50)
    def load_resnet(self, sd: Dict[str, torch.Tensor], arch: str, prefix: str = '') -> None:
        """Hand a ``resnet_backbone.<arch>()`` state dict to the library: select the arch, then its conv+BN pairs in
        state-dict order and the four Linear heads concatenated in the reference's output order ori | shape | exp | tex
        (resnet_backbone.py:242-246)."""
        if arch not in RESNET_ARCHS:
            raise RuntimeError(f"arch '{arch}': the ResNet backbones are {', '.join(RESNET_ARCHS)}")
        feat = 512 if RESNET_ARCHS[arch][0] < 50 else 2048
        self._load_convbn('resnet', arch, ('syn_resnet_select', *RESNET_ARCHS[arch]), resnet_conv_keys(arch), feat, sd, prefix)

    def load_resnet50(self, sd: Dict[str, torch.Tensor], prefix: str = '') -> None:
        """Hand a ``resnet_backbone.resnet50()`` state dict to the library (53 conv+BN pairs in execution order, the four
        Linear heads concatenated in the reference's output order ori | shape | exp | tex, resnet_backbone.py:242-246)."""
        self.load_resnet(sd, 'resnet50', prefix)

    @property
    def resnet_feature_dim(self) -> int:
        """Pooled feature width of the selected ResNet: 512 (resnet18 / 34) or 2048."""
        return self._backbone('resnet')[1]

    def forward_resnet(self, x: torch.Tensor):
        """ResNet._forward_impl (resnet_backbone.py:227-249) of the loaded arch: (B,3,120,120) fp32 normalised crops or raw
        uint8 crops -> ((B,102) ori|shape|exp|tex, (B,512 or 2048) pooled)."""
        return self._forward_convbn('resnet', x)

    def forward_resnet50(self, x: torch.Tensor):
        """ResNet._forward_impl (resnet_backbone.py:227-249): (B,3,120,120) -> ((B,102) ori|shape|exp|tex, (B,2048) pooled)."""
        x = self._check_x(x)
        b = x.shape[0]
        out = torch.empty((b, 102), device=self.device, dtype=torch.float32)
        pool = torch.empty((b, 2048), device=self.device, dtype=torch.float32)
        self._call('syn_resnet50_forward', x.data_ptr(), b, out.data_ptr(), pool.data_ptr())
        return out, pool

    def debug_resnet_until(self, x: torch.Tensor, stage: int):
        """Run of the loaded ResNet up to ``stage`` (0 stem, 1 max-pool, 1 + i conv i of the plan, n + 1 avgpool, n + 2
        heads, n convs; 54 / 55 for resnet50): (that stage's output as (rows, channels) -- one row per NHWC pixel, or per
        face --, its row maxima as int32 fp32 bit patterns, or None for a stage that records none)."""
        x = self._check_x(x)
        b = x.shape[0]
        arch, feat = self._backbone('resnet')
        keys = resnet_conv_keys(arch)
        n = len(keys)
        if stage == 0:
            rows, cols, rm = b * 3600, 64, True
        elif stage == 1:
            rows, cols, rm = b * 900, 64, True
        elif stage <= n:
            d = _lib.ConvDesc()
            _lib.check(self._lib.syn_resnet_arch_conv_desc(*RESNET_ARCHS[arch], stage - 1, C.byref(d)))
            rows, cols, rm = b * d.h_out * d.h_out, d.cout, 'downsample' not in keys[stage - 1][0]
        else:
            rows, cols, rm = b, feat if stage == n + 1 else 102, stage == n + 1
        return self._debug_run('syn_debug_resnet_until', x, stage, rows, cols, rm)

    # MobileNetV1 backbones (backbone_nets/mobilenetv1_backbone.py, the five mobilenet_* factories)
    def load_mobilenet_v1(self, sd: Dict[str, torch.Tensor], arch: str, prefix: str = '') -> None:
        """Hand a ``mobilenetv1_backbone.<arch>()`` state dict to the library (27 conv+BN pairs in execution order, the four
        Linear heads concatenated in the reference's output order ori | shape | exp | tex, mobilenetv1_backbone.py:132-138)."""
        if arch not in MBV1_WIDTHS:
            raise RuntimeError(f"arch '{arch}': MobileNetV1 widths are {', '.join(MBV1_WIDTHS)}")
        code = int(round(MBV1_WIDTHS[arch] * 100))
        self._load_convbn('mbv1', arch, ('syn_mbv1_set_widen', code), mobilenet_v1_conv_keys(), 1024 * code // 100, sd, prefix)

    def forward_mobilenet_v1(self, x: torch.Tensor):
        """MobileNet.forward (mobilenetv1_backbone.py:108-140): (B,3,120,120) fp32 normalised crops or raw uint8 crops ->
        ((B,102) ori|shape|exp|tex, (B,1024w) pooled)."""
        return self._forward_convbn('mbv1', x)

    def debug_mobilenet_v1_until(self, x: torch.Tensor, stage: int):
        """MobileNetV1 run up to ``stage`` (0 stem, 2j - 1 / 2j conv_dw / conv_sep of block j = 1..13, 27 avgpool, 28
        heads): (that stage's output as (rows, channels) -- one row per NHWC pixel, or per face --, its row maxima as int32
        fp32 bit patterns, or None for a stage that records none)."""
        x = self._check_x(x)
        b = x.shape[0]
        arch, feat = self._backbone('mbv1')
        if stage <= 26:
            d = _lib.ConvDesc()
            _lib.check(self._lib.syn_mbv1_conv_desc(int(round(MBV1_WIDTHS[arch] * 100)), stage, C.byref(d)))
            rows, cols, rm = b * d.h_out * d.h_out, d.cout, stage == 0 or stage % 2 == 1 or stage == 26
        else:
            rows, cols, rm = b, feat if stage == 27 else 102, stage == 27
        return self._debug_run('syn_debug_mbv1_until', x, stage, rows, cols, rm)

    # GhostNet backbone (backbone_nets/ghostnet_backbone.py, ghostnet() at width 1.0)
    def load_ghostnet(self, sd: Dict[str, torch.Tensor], prefix: str = '') -> None:
        """Hand a ``ghostnet_backbone.ghostnet()`` state dict to the library: its 95 convs in state-dict order (conv+BN
        pairs, and the SE convs and conv_head with their biases), the four Linear heads concatenated in the reference's
        output order ori | shape | exp | tex (ghostnet_backbone.py:229-233), then commit."""
        with self._lock:
            self._backbones['ghost'] = ('ghostnet', 1280)
            for i, (ck, bk) in enumerate(ghostnet_conv_keys()):
                w = _host_f32(sd[f'{prefix}{ck}.weight'])
                if bk is None:
                    b = _host_f32(sd[f'{prefix}{ck}.bias'])
                    self._call_host('syn_ghost_set_conv_bias', i, w.data_ptr(), w.numel(), b.data_ptr())
                else:
                    bn = [_host_f32(sd[f'{prefix}{bk}.{k}']) for k in ('weight', 'bias', 'running_mean', 'running_var')]
                    self._call_host('syn_ghost_set_conv', i, w.data_ptr(), w.numel(), *[t.data_ptr() for t in bn], 1e-5)
            w = torch.cat([_host_f32(sd[f'{prefix}{k}.weight']) for k in GHOSTNET_HEADS]).contiguous()
            b = torch.cat([_host_f32(sd[f'{prefix}{k}.bias']) for k in GHOSTNET_HEADS]).contiguous()
            if tuple(w.shape) != (102, 1280):
                raise RuntimeError(f'ghostnet heads: expected (102, 1280) weights, got {tuple(w.shape)}')
            self._call_host('syn_ghost_set_heads', w.data_ptr(), b.data_ptr())
            self._call_host('syn_ghost_commit')

    def forward_ghostnet(self, x: torch.Tensor):
        """GhostNet.forward (ghostnet_backbone.py:214-233) in eval mode: (B,3,120,120) fp32 normalised crops or raw uint8
        crops -> ((B,102) ori|shape|exp|tex, (B,1280) the conv_head output after its ReLU, which the heads read)."""
        return self._forward_convbn('ghost', x)

    def ghostnet_stage_desc(self, stage: int) -> Tuple[int, int, bool]:
        """(rows per face, columns, records row maxima) of stage ``stage`` of debug_ghostnet_until."""
        r, c, m = C.c_int(0), C.c_int(0), C.c_int(0)
        _lib.check(self._lib.syn_ghost_stage_desc(int(stage), C.byref(r), C.byref(c), C.byref(m)))
        return r.value, c.value, bool(m.value)

    def debug_ghostnet_until(self, x: torch.Tensor, stage: int):
        """GhostNet run up to ``stage`` (one stage per launch output, include/synergy_b200.h syn_debug_ghost_until):
        (that stage's output as (rows, channels) -- one row per NHWC pixel, or per face --, its row maxima as int32 fp32
        bit patterns, or None for a stage that records none)."""
        x = self._check_x(x)
        self._backbone('ghost')
        rows, cols, rm = self.ghostnet_stage_desc(stage)
        return self._debug_run('syn_debug_ghost_until', x, stage, x.shape[0] * rows, cols, rm)

    # ---- per-stage debug runs of the GEMM layers (include/synergy_b200.h syn_debug_*_until / syn_debug_gemm) ----
    RESNET_STAGES = 56
    FOR_STAGES = ((64, True), (64, True), (64, True), (128, True), (1024, False), (1024, False), (2360, True),
                  (512, False), (512, True), (256, True), (128, True), (3, False), (3 * 68, False))   # (columns, row maxima)
    REV_STAGES = FOR_STAGES[:5] + ((1024, True), (N_PARAMS, False))

    def _debug_out(self, rows: int, cols: int, rowmax: bool):
        out = torch.empty((rows, cols), device=self.device, dtype=torch.float32)
        rm = torch.zeros((rows,), device=self.device, dtype=torch.int32) if rowmax else None
        return out, rm

    def debug_pointnet_until(self, net: int, lmk: torch.Tensor, stage: int, pool: Optional[torch.Tensor] = None,
                             params: Optional[torch.Tensor] = None):
        """MLP_for (net 0) or MLP_rev (net 1) run up to ``stage`` (include/synergy_b200.h): (output (rows, columns),
        row maxima as int32 fp32 bit patterns or None).  Rows are the B*68 points, point-major, or the B faces."""
        lmk = self._dev_f32(lmk)
        b = lmk.shape[0]
        cols, rm = (self.FOR_STAGES if net == 0 else self.REV_STAGES)[stage]
        per_face = stage >= 5 and not (net == 0 and 8 <= stage <= 11)
        out, rmax = self._debug_out(b if per_face else b * 68, cols, rm)
        pool = self._dev_f32(pool) if pool is not None else None
        params = self._dev_f32(params) if params is not None else None
        self._call('syn_debug_pointnet_until', net, lmk.data_ptr(), pool.data_ptr() if pool is not None else None,
                   params.data_ptr() if params is not None else None, b, stage, out.data_ptr(), rmax.data_ptr() if rm else None)
        return out, rmax

    def debug_gemm(self, w: torch.Tensor, bias: torch.Tensor, a: torch.Tensor, rowmax_in: torch.Tensor, act: int = 0,
                   conv: Optional[Tuple[int, int, int, int, int]] = None, residual: Optional[torch.Tensor] = None,
                   addend: Optional[torch.Tensor] = None, addend_group: int = 1, colmax_group: int = 0):
        """One tc_gemm_kernel launch on a layer built from ``w`` (N, K) and ``bias`` (N,).  ``a``: (M, lda) rows, or NHWC
        maps when ``conv`` = (ksize, stride, pad, HO, WO); ``rowmax_in``: int32 fp32 bit patterns per row / input pixel.
        act 0 none, 2 ReLU.  colmax_group > 0 also max-pools the output over groups of that many rows.
        Returns (out (M, N), rowmax_out (M,) int32 bits, colmax (ceil(M / group), N) int32 bits or None)."""
        w, bias = _host_f32(w), _host_f32(bias)
        n, k = w.shape
        a = self._dev_f32(a)
        if conv is None:
            m, lda, ks, st, pad, hh, ww, cc = a.shape[0], a.shape[1], 0, 1, 0, 0, 0, 0
        else:
            ks, st, pad, ho, wo = conv
            bb, hh, ww, cc = a.shape
            m, lda = bb * ho * wo, cc
        out = torch.empty((m, n), device=self.device, dtype=torch.float32)
        rmo = torch.zeros((m,), device=self.device, dtype=torch.int32)
        cm = torch.zeros((-(-m // colmax_group), n), device=self.device, dtype=torch.int32) if colmax_group > 0 else None
        rmi = rowmax_in.to(device=self.device, dtype=torch.int32).contiguous()
        res = self._dev_f32(residual) if residual is not None else None
        add = self._dev_f32(addend) if addend is not None else None
        ptr = lambda t: t.data_ptr() if t is not None else None
        self._call('syn_debug_gemm', w.data_ptr(), bias.data_ptr(), n, k, act, ks, st, pad, hh, ww, cc, a.data_ptr(), m, lda,
                   rmi.data_ptr(), ptr(res), ptr(add), addend_group, ptr(cm), colmax_group, out.data_ptr(), rmo.data_ptr())
        return out, rmo, cm

    # ---- poisoned workspaces (tests only, include/synergy_b200.h syn_debug_fill_workspaces) ------------------------
    def debug_fill_workspaces(self, byte: int) -> int:
        """Set every byte of every device workspace the handle has grown, at its allocated size, to ``byte``, ordered
        on the current stream after the previous call; returns the number of bytes filled."""
        n = C.c_size_t(0)
        self._call('syn_debug_fill_workspaces', int(byte), C.byref(n))
        return int(n.value)

    def debug_fill_on_grow(self, byte: int) -> None:
        """Every later workspace growth sets its new buffers to ``byte`` (-1: off)."""
        self._call_host('syn_debug_fill_on_grow', int(byte))

    def debug_forward_until(self, x: torch.Tensor, layer: int) -> torch.Tensor:
        x = self._check_x(x)
        spec = conv_plan()[layer]
        out = torch.empty((x.shape[0], spec.h_out, spec.h_out, spec.cout), device=self.device, dtype=torch.float32)
        self._call('syn_debug_forward_until', x.data_ptr(), x.shape[0], layer, out.data_ptr())
        return out
