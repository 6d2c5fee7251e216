import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on the H100 box)')


@pytest.fixture(scope='session')
def synth_pack():
    """Seeded synthetic 3DMM, shared by every test (32 MB, built once)."""
    from synergynet_b200 import synthetic
    from synergynet_b200.params import ParamsPack, set_param_pack
    pack = ParamsPack(arrays=synthetic.make_3dmm(seed=0))
    set_param_pack(pack)
    return pack
