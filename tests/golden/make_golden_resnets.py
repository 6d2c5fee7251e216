#!/usr/bin/env python
"""Generate ``tests/golden/ref_vectors_resnets.npz`` by running the UNMODIFIED reference ResNet backbones on the CPU
(fp32), in the same scratch copy of the reference tree as ``make_golden.py`` (needs the reference checkout):

    python tests/golden/make_golden_resnets.py

For each of the six ResNet factories other than resnet50 (whose vectors are in ``ref_vectors.npz``;
resnet_backbone.py:282-391): the seeded checkpoint of ``oracle/synth_resnet.py`` is loaded with ``strict=True``, the
module's own forward runs on four seeded structured crops, and ``out102`` and the adapter's landmarks (the reference's
``reconstruct_vertex_62`` of ``out102[:, :62]``) are recorded, together with the reference's state_dict key list.  Inputs
and weights are regenerated from their seeds by the tests; only outputs and key names are stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from synergynet_b200 import synthetic  # noqa: E402
from synergynet_b200.backbone import RESNET_ARCHS  # noqa: E402
from oracle import synth_resnet  # noqa: E402
from make_golden import scratch_reference  # noqa: E402

OUT = os.path.join(HERE, 'ref_vectors_resnets.npz')
FACES, CROP_SEED = 4, 31
ARCHS = tuple(a for a in RESNET_ARCHS if a != 'resnet50')


def crops_u8():
    return synthetic.make_structured_crops_u8(FACES, seed=CROP_SEED)


def main():
    torch.manual_seed(0)
    sds = {arch: synth_resnet.build_resnet_state_dict(0, arch) for arch in ARCHS}
    scratch_reference()
    import synergy3DMM as ref_api                    # the reference modules, unmodified
    from backbone_nets import resnet_backbone as ref_resnet
    ref = ref_api.SynergyNet()
    ref.eval()
    x = synthetic.normalize_crops(crops_u8())
    out = {}
    for arch, sd in sds.items():
        net = getattr(ref_resnet, arch)(pretrained=False)
        res = net.load_state_dict(sd, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        net.eval()
        with torch.no_grad():
            o = net(x)
            lmk = ref.reconstruct_vertex_62(o[:, :62].contiguous(), dense=False)
        assert float(o.std(dim=0).min()) > 1e-3, f'{arch}: the faces give the same output'
        out[f'{arch}_out102'] = o.numpy()
        out[f'{arch}_lmk'] = lmk.numpy()
        out[f'{arch}_keys'] = np.array(list(net.state_dict().keys()))
    out['meta'] = np.array([f'torch={torch.__version__}', 'reference=choyingw/SynergyNet@9de11e2', 'checkpoint seed=0',
                            f'crops=make_structured_crops_u8({FACES}, seed={CROP_SEED})'])
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
