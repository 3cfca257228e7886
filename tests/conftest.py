import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need a CUDA device: skip (not fail) them where none is visible (the CPU container)."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:   # noqa: BLE001
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="no CUDA device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name_prefix):
    """Golden vectors produced by the unmodified reference (tests/golden/generate.py)."""
    for fn in sorted(os.listdir(GOLDEN_DIR)):
        if fn.startswith(name_prefix) and fn.endswith(".npz"):
            z = np.load(os.path.join(GOLDEN_DIR, fn))
            n = int(z["n_params"])
            return dict(coords=z["coords"], u=z["u"], residual=z["residual"], loss=float(z["loss"]),
                        residual32=z["residual32"], loss32=float(z["loss32"]),
                        params=[z[f"param_{i}"] for i in range(n)], grads=[z[f"grad_{i}"] for i in range(n)],
                        grads32=[z[f"grad32_{i}"] for i in range(n)])
    raise FileNotFoundError(name_prefix)


@pytest.fixture(autouse=True)
def _seed():
    import torch
    torch.manual_seed(42)
    np.random.seed(42)
