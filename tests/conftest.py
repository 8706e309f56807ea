import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (the project targets the H100, sm_90a)")
    config.addinivalue_line("markers", "slow: minutes of host work (10 M-triangle scene build); runs only with RT_TEST_SLOW=1")


def pytest_collection_modifyitems(config, items):
    if os.environ.get("RT_TEST_SLOW"):
        return
    skip = pytest.mark.skip(reason="slow: set RT_TEST_SLOW=1")
    for item in items:
        if "slow" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(REPO, "tests", "golden")
