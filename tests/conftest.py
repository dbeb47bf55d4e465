import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


def pytest_collection_modifyitems(config, items):
    """Tests that execute the reference's own GPU binaries (oracle/_ref/ref_harness_gpu: cuBLAS + cuSPARSE) go last:
    on a freshly provisioned box the first load of those libraries has been seen to take minutes."""
    slow = [it for it in items if "reference_driver" in it.name or "reference_amr" in it.name]
    if slow:
        items[:] = [it for it in items if it not in slow] + slow


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def penal_golden():
    """(L, steps) of tests/golden/penal_L4.npz: the reference's penalisation phase, recorded step by step"""
    sys.path.insert(0, GOLDEN)
    from make_golden import load_penal
    return load_penal(os.path.join(GOLDEN, "penal_L4.npz"))
