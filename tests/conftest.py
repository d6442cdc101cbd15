import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLD = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def sds():
    from oracle.weights import make_state_dict

    return {k: make_state_dict(k, seed=0) for k in ("vgg", "warp", "color")}


@pytest.fixture(scope="session")
def ctx(sds):
    """Shared libdvc context with the seeded weights loaded (GPU tests only)."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import dvc

    c = dvc.get_context(0)
    c.set_weights(dvc.NET_VGG, sds["vgg"])
    c.set_weights(dvc.NET_WARP, sds["warp"])
    c.set_weights(dvc.NET_COLOR, sds["color"])
    if os.environ.get("DVC_TEST_KC"):  # parity of a coarser accumulator promotion chunk (conv_tc.cu)
        c.debug_flag("tc_kc", int(os.environ["DVC_TEST_KC"]))
    return c


def load_golden(name):
    import numpy as np

    return dict(np.load(os.path.join(GOLD, name + ".npz")))
