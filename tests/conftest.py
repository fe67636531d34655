"""pytest config: registers the `gpu` marker and puts the repo root on sys.path.

`-m "not gpu"` : oracle vs golden vectors, host logic, C-ABI symbol checks (CPU only).
`-m gpu`       : parity tests proper -- CUDA path through the C-ABI vs the oracle.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def golden():
    import json

    with open(os.path.join(ROOT, "tests", "golden", "reference_cases.json")) as f:
        return json.load(f)
