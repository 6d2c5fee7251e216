"""Drop-in twin of the reference pip-style API ``synergy3DMM.SynergyNet()``
(reference synergy3DMM.py:70-207): no-argument constructor, MobileNetV2 fixed, weights looked up
in ``pretrained/best.pth.tar`` next to the package (load errors swallowed like the reference,
:109-113), ``.eval()``; ``forward_test`` / ``reconstruct_vertex_62`` / ``get_all_outputs`` run on
the sm_90a library."""
from __future__ import annotations

import os
import types

from .model_building import I2P, _SynergyBase, parse_param_62  # noqa: F401
from .params import get_param_pack

prefix_path = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


class SynergyNet(_SynergyBase):
    def __init__(self):
        super().__init__()
        args = types.SimpleNamespace(arch='mobilenet_v2',
                                     checkpoint_fp=os.path.join(prefix_path, 'pretrained/best.pth.tar'))
        self._setup(args, get_param_pack(), None)
        try:
            print('loading weights from ', args.checkpoint_fp)
            self.load_weights(args.checkpoint_fp)
        except Exception:
            pass
        self.eval()
