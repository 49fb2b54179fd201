import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "raft-ncup_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


@pytest.fixture(scope="session")
def gold():
    z = np.load(os.path.join(ROOT, "tests", "golden", "cfg1.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


@pytest.fixture(scope="session")
def meta():
    with open(os.path.join(ROOT, "tests", "golden", "meta.json")) as f:
        return json.load(f)


from rnc.synth import build_model, frames, ref_args  # noqa: E402,F401  (shared with bench.py)


@pytest.fixture(scope="session")
def sd_ncup():
    return {k: v.detach() for k, v in build_model("raft_nc_dbl").state_dict().items()}


@pytest.fixture(scope="session")
def sd_raft():
    return {k: v.detach() for k, v in build_model("raft").state_dict().items()}
