import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def built():
    """Build the CUDA library, the hetmers executable and the oracle once per session."""
    import __graft_entry__ as ge
    ge.build()
    return True


@pytest.fixture(scope="session")
def golden_meta():
    import json
    with open(os.path.join(GOLDEN, "golden.json")) as f:
        return json.load(f)


def golden_cases():
    import json
    with open(os.path.join(GOLDEN, "golden.json")) as f:
        return sorted(k for k in json.load(f) if not k.startswith("_"))
