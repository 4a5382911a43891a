import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "pytorch-r2d2-dpg_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """Fixture `name`; a large one is stored as <stem>.part0.npz, <stem>.part1.npz, ... (oracle/make_golden.py)."""
    stem = name[:-len(".npz")]
    parts = sorted((f for f in os.listdir(GOLDEN) if f.startswith(stem + ".part") and f.endswith(".npz")),
                   key=lambda f: int(f[len(stem) + 5:-4]))
    out = {}
    for f in parts or [name]:
        z = np.load(os.path.join(GOLDEN, f), allow_pickle=False)
        out.update({k: z[k] for k in z.files})
    return out


def golden_params(g, prefix):
    """{'l1.weight': ...} for keys 'prefix/<key>'."""
    n = len(prefix) + 1
    return {k[n:]: v for k, v in g.items() if k.startswith(prefix + "/")}


def golden_batch(g, it):
    return {k: g[f"it{it}/{k}"] for k in ("obs", "act", "rew", "term", "a_state", "ta_state", "c_state", "tc_state")}


def rel_l2(a, b):
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))
