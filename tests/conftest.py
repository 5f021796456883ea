import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_package():
    return importlib.import_module("monte-carlo-ray-tracer_b200")


@pytest.fixture(scope="session")
def mcrt():
    return load_package()


def golden_cases():
    return sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz") and not f.endswith("_kat.npz"))
