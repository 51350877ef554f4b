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
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")
    config.addinivalue_line("markers", "needs_reference: needs /root/reference (build container only)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """tests/golden/<name>.npz -> dict of torch tensors (+ 'sd' sub-dict, 'grad' sub-dict)."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    out, sd, grad = {}, {}, {}
    for k in z.files:
        v = z[k]
        if k == "__meta__" or k == "kw":
            out[k] = str(v)
            continue
        t = torch.from_numpy(np.ascontiguousarray(v))
        if k.startswith("sd/"):
            sd[k[3:]] = t
        elif k.startswith("grad/"):
            grad[k[5:]] = t
        else:
            out[k] = t
    out["sd"], out["grad"] = sd, grad
    if "kw" in out:
        out["kw"] = eval(out["kw"], {"__builtins__": {}}, {})  # repr of a plain dict of literals
    return out


def rel_err(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30))


@pytest.fixture(scope="session")
def golden():
    return load_golden
