"""pytest config: the `gpu` marker + import paths.

`-m "not gpu"` runs without a GPU (oracle vs golden vectors, host logic, C-ABI symbol
check); `-m gpu` needs an H100 and calls through the C-ABI library."""
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "normalizing-flows_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: the library is built for sm_90a)")


def load_golden(name):
    """-> (spec, sd, arrays) from tests/golden/<name>.npz (minted from the reference).  A golden whose weights are too
    large to store carries a rebuild recipe and digests instead (tests/helpers.py state_dict_from_recipe)."""
    f = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    if "sd_recipe" in f.files:
        from helpers import state_dict_from_recipe
        sd = state_dict_from_recipe(json.loads(str(f["sd_recipe"])), json.loads(str(f["sd_sha256"])))
    else:
        sd = {k[4:]: f[k] for k in f.files if k.startswith("sd__")}
    spec = json.loads(str(f["spec"])) if "spec" in f.files else None
    arr = {k: f[k] for k in f.files if not k.startswith("sd__") and k not in ("spec", "sd_recipe", "sd_sha256")}
    return spec, sd, arr


@pytest.fixture(scope="session")
def golden():
    return load_golden


@pytest.fixture(autouse=True)
def _no_grad_by_default():
    """The parity tests exercise the density pass; gradient tests opt in with torch.enable_grad()."""
    import torch
    prev = torch.is_grad_enabled()
    torch.set_grad_enabled(False)
    yield
    torch.set_grad_enabled(prev)
