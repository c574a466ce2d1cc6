"""pytest configuration: registers the `gpu` marker and puts the repo root on sys.path.

`-m "not gpu"` runs on the build container (no GPU): oracle-vs-golden, host logic, C-ABI symbol checks, gloo tests.
`-m gpu` runs on an H100: parity of the CUDA path (through the C-ABI) against the oracle.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
