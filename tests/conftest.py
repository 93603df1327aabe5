"""Test configuration.

`-m "not gpu"` covers the oracle against the golden vectors, the host logic
through the C ABI, and that the library loads and exports every declared
symbol.  `-m gpu` holds the parity tests proper (CUDA path vs oracle).
"""
import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the C-ABI library and the C oracle once (cross-compiles without a GPU)."""
    import __graft_entry__ as g
    g.build()


@pytest.fixture(scope="session")
def cro(_built):
    return importlib.import_module("composable-resource-operator_b200")


@pytest.fixture(scope="session")
def oracle(_built):
    import oracle as o
    return o


@pytest.fixture(scope="session")
def coracle(oracle):
    return oracle.COracle()


@pytest.fixture(scope="session")
def kats():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "reference_kats.json")) as f:
        return json.load(f)
