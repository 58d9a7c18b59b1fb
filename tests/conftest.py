import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90a)")


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "reference_vectors.json")) as f:
        return json.load(f)


def rust_debug_f64(x):
    """Rust `{:?}` for f64 in the value range of the fixtures (shortest round-trip, '.0' suffix)."""
    return repr(float(x))


@pytest.fixture(scope="session")
def fmt_f64():
    return rust_debug_f64
