import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def golden_names(prefix):
    return sorted(f[:-4] for f in os.listdir(GOLDEN_DIR)
                  if f.startswith(prefix) and f.endswith(".npz"))


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN_DIR
