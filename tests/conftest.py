import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import binding
    binding.lib()
    return binding


@pytest.fixture(scope="session")
def fixture_map():
    d = np.load(os.path.join(ROOT, "tests", "golden", "fixture_gridmap.npz"))
    m = json.load(open(os.path.join(ROOT, "tests", "golden", "fixture_gridmap.json")))
    return m, {k: np.asfortranarray(d[k]) for k in d.files}


@pytest.fixture(scope="session")
def te():
    import traversability_estimation_b200 as mod
    return mod


@pytest.fixture(scope="session")
def ctx(te):
    c = te.Context(0)
    yield c
    c.close()
