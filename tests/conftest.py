import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a; run with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(autouse=True)
def _no_workers_left_behind():
    """Multi-process tests spawn gloo workers.  When one of them fails, its peers may sit in a collective for minutes; left
    alive they load the host and make the tests that follow time out in turn.  Whatever a test leaves behind is terminated
    here."""
    yield
    import multiprocessing
    for p in multiprocessing.active_children():
        p.terminate()
    for p in multiprocessing.active_children():
        p.join(5)
