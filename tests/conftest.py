import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()

import torch  # noqa: E402

torch.set_num_threads(min(16, os.cpu_count() or 1))  # the CPU oracle oversubscribes badly on 128-core hosts

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
