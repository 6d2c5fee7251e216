#!/usr/bin/env python
"""Generate ``tests/golden/ref_vectors_ghostnet.npz`` by running the UNMODIFIED reference GhostNet backbone on the CPU
(fp32, eval mode), in the same scratch copy of the reference tree as ``make_golden.py`` (needs the reference checkout):

    python tests/golden/make_golden_ghostnet.py

The seeded calibrated checkpoint of ``oracle/synth_ghost.py`` is loaded into ``ghostnet_backbone.ghostnet()`` with
``strict=True``, the module's own forward runs on four seeded structured crops, and ``out102`` is recorded together with
the reference's state_dict key list.  Inputs and weights are regenerated from their seeds by the tests; only outputs and
key names are stored.
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
from oracle import synth_ghost  # noqa: E402
from make_golden import scratch_reference  # noqa: E402

OUT = os.path.join(HERE, 'ref_vectors_ghostnet.npz')
FACES, CROP_SEED = 4, 31


def main():
    torch.manual_seed(0)
    sd = synth_ghost.build_ghostnet_state_dict(0)
    scratch_reference()
    from backbone_nets import ghostnet_backbone as ref_ghost        # the reference module, unmodified
    net = ref_ghost.ghostnet()
    res = net.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    net.eval()
    x = synthetic.normalize_crops(synthetic.make_structured_crops_u8(FACES, seed=CROP_SEED))
    with torch.no_grad():
        o = net(x)
    assert float(o.std(dim=0).min()) > 1e-3, 'the faces give the same output'
    out = {'ghostnet_out102': o.numpy(), 'ghostnet_keys': np.array(list(net.state_dict().keys())),
           'meta': np.array([f'torch={torch.__version__}', 'reference=choyingw/SynergyNet@9de11e2', 'checkpoint seed=0',
                             f'crops=make_structured_crops_u8({FACES}, seed={CROP_SEED})'])}
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
