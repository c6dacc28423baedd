import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


class Golden:
    """One tests/golden/*.npz fixture: cfg (dict) + arrays; helpers to pull
    prefixed groups out as torch tensors."""

    def __init__(self, name):
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        self.cfg = json.loads(bytes(z["cfg"]).decode())
        self.arrays = {k: z[k] for k in z.files if k != "cfg"}

    def t(self, key, device="cpu"):
        return torch.from_numpy(np.array(self.arrays[key])).to(device)

    def group(self, prefix, device="cpu"):
        return {k[len(prefix):]: torch.from_numpy(np.array(v)).to(device)
                for k, v in self.arrays.items() if k.startswith(prefix)}


@pytest.fixture(scope="session")
def golden():
    cache = {}

    def load(name):
        if name not in cache:
            cache[name] = Golden(name)
        return cache[name]

    return load


def rel_l2(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))
