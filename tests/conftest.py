import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
CONV_FIXTURES = ["c1_norte", "c1_rte", "rand_t3r4_dk4", "rand_dk25", "mag_mini_dk50", "oag_mini", "hub_h2"]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100 / sm_90a)")


def load_golden(name):
    """tests/golden/<name>.pt, merged with its <name>.part<i>.pt files (oracle/make_golden.py:save_fixture splits a
    fixture's top-level entries over several files so that none passes 1 MB)."""
    import glob
    import torch
    fx = torch.load(os.path.join(GOLDEN_DIR, name + ".pt"), map_location="cpu", weights_only=False)
    parts = glob.glob(os.path.join(glob.escape(GOLDEN_DIR), glob.escape(name) + ".part*.pt"))
    for path in sorted(parts, key=lambda p: int(p.rsplit(".part", 1)[1][:-3])):
        fx.update(torch.load(path, map_location="cpu", weights_only=False))
    return fx


def load_golden_json(name):
    import json
    with open(os.path.join(GOLDEN_DIR, name + ".json")) as f:
        return json.load(f)


@pytest.fixture(params=CONV_FIXTURES)
def conv_fixture(request):
    fx = load_golden(request.param)
    fx["name"] = request.param
    return fx
