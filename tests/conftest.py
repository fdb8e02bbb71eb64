import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) GPU; select with -m gpu")


@pytest.fixture(scope="session")
def golden_dir():
    return ROOT / "tests" / "golden"


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """The C-ABI library must exist for every test (symbols on CPU, kernels on GPU); build it once if absent."""
    from mimo_b200 import build
    build.build()
