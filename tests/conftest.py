import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def pkg():
    import pcnn_loader
    return pcnn_loader.load()


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    import json
    g = os.path.join(ROOT, "tests", "golden")
    out = dict(np.load(os.path.join(g, "mnist_subset.npz")))
    out.update(dict(np.load(os.path.join(g, "reference_vectors.npz"))))
    out["scalars"] = json.load(open(os.path.join(g, "reference_scalars.json")))
    return out


@pytest.fixture(scope="session")
def eng(pkg):
    """One engine for the GPU session; fails loudly (no skip, no fallback) if the CUDA library cannot run."""
    e = pkg.Engine(0)
    yield e
    e.close()
