import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "warp-transducer_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests are skipped (not failed) on a host without a CUDA device."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def known_answers():
    import json
    return json.load(open(os.path.join(GOLDEN, "known_answers.json")))


@pytest.fixture(scope="session")
def ref_cases():
    z = np.load(os.path.join(GOLDEN, "ref_cases.npz"))
    cases = {}
    for name in z["names"]:
        name = str(name)
        cases[name] = {k.split(".", 1)[1]: z[k] for k in z.files if k.startswith(name + ".")}
    return cases
