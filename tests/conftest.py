"""pytest configuration: `gpu` marker + import paths.

`-m "not gpu"` covers the oracle against the reference's known-answer vectors, host logic and the
C-ABI symbol surface; `-m gpu` are the parity tests proper (CUDA path vs oracle through the C ABI).
"""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
if str(ROOT / "tests") not in sys.path:
    sys.path.insert(0, str(ROOT / "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


@pytest.fixture(scope="session")
def hxo():
    from oracle import hxo as m

    m.build()
    return m
