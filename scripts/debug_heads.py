#!/usr/bin/env python
"""Stage-by-stage comparison of MLP_for on the GPU against the CPU oracle (debug aid, needs an H100)."""
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import reference_port as rp, synth_model  # noqa: E402
from synergynet_b200 import _lib, model_building, synthetic  # noqa: E402
from synergynet_b200.params import ParamsPack, set_param_pack  # noqa: E402


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def main():
    set_param_pack(ParamsPack(arrays=synthetic.make_3dmm(seed=0)))
    sd = synth_model.build_state_dict(0)
    basis = rp.gather_sparse_basis(synthetic.make_3dmm(0))
    m = model_building.SynergyNet(types.SimpleNamespace(arch='mobilenet_v2', img_size=120, devices_id=[0]))
    m.load_state_dict(sd, strict=True)
    m.eval()
    B = 5
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(B, seed=71))
    attr, pool = rp.mobilenetv2_forward(sd, x)
    lmk = torch.from_numpy(rp.reconstruct_vertex_62(attr.numpy(), basis))
    pre = 'forwardDirection.'
    s = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
    L = lambda t, i: rp._pn_layer(s, t, f'conv{i}', f'bn{i}')
    o1 = L(lmk, 1); pf = L(o1, 2); o3 = L(pf, 3); o4 = L(o3, 4); o5 = L(o4, 5)
    glob = F.max_pool1d(o5, 68)
    rep = lambda t: t.unsqueeze(2).repeat(1, 1, 68) if t.dim() == 2 else t.repeat(1, 1, 68)
    cat = torch.cat([pf, rep(glob), rep(pool), rep(attr[:, 12:52]), rep(attr[:, 52:62])], 1)
    o6 = L(cat, 6); o7 = L(o6, 7); o8 = L(o7, 8); o9 = L(o8, 9)
    eng = m._pointnet_engine(x.cuda(), 0)
    res, ref = eng.mlp_for(lmk.cuda(), pool.cuda(), attr.cuda())
    lib = _lib.load()

    def buf(which, n):
        out = torch.empty(n, dtype=torch.float32)
        _lib.check(lib.syn_debug_heads_buffer(eng._h, which, out.data_ptr(), n))
        return out.numpy()
    M = B * 68
    pm = lambda t: t.permute(0, 2, 1).reshape(M, -1).numpy()           # (B,C,68) -> point-major rows
    print('point_features   ', rel(buf(0, M * 64).reshape(M, 64), pm(pf)))
    print('global max-pool  ', rel(buf(5, B * 1024).reshape(B, 1024), glob[:, :, 0].numpy()))
    fv = buf(1, B * 2360).reshape(B, 2360)
    want_fv = torch.cat([glob[:, :, 0], pool, attr[:, 12:62]], 1).numpy()
    print('face vector      ', rel(fv[:, :2354], want_fv), 'pad', float(np.abs(fv[:, 2354:]).max()))
    # conv6 face part: BN-folded weights columns 64..2418 times the face vector (no bias)
    w6 = s['conv6.weight'][:, :, 0].double(); sc = (s['bn6.weight'].double() / torch.sqrt(s['bn6.running_var'].double() + 1e-5))
    face = (torch.from_numpy(want_fv).double() @ (w6[:, 64:] * sc[:, None]).T).float().numpy()
    print('conv6 face part  ', rel(buf(2, B * 512).reshape(B, 512), face))
    print('conv8 out (bufA) ', rel(buf(3, M * 128).reshape(M, 128), pm(o8)))
    print('conv9 out (bufB) ', rel(buf(4, M * 3).reshape(M, 3), pm(o9)))
    print('residual         ', rel(res.cpu().numpy(), o9.numpy()), 'refined', rel(ref.cpu().numpy(), (lmk + 0.05 * o9).numpy()))
    print('oracle conv6/7 stats', float(o6.abs().max()), float(o7.abs().max()), float(o9.abs().max()))
    rev = m._pointnet_engine(x.cuda(), 1).mlp_rev((lmk + 0.05 * o9).cuda())
    print('mlp_rev          ', rel(rev.cpu().numpy(), rp.mlp_rev_forward(sd, lmk + 0.05 * o9).numpy()))
    loss = m(x.cuda(), (attr + 0.1).cuda())
    lo, _ = rp.synergy_forward(sd, basis, x, attr + 0.1)
    for k in lo:
        print(k, rel(loss[k].cpu().numpy(), lo[k].numpy()))


if __name__ == '__main__':
    main()
