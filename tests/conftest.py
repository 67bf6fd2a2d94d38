import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "late: run after every other test (cases added after the last GPU visit)")


# Streams of the first GPU visits; the feature streams added after the last visit are pinned on the CPU only so far
# (tests/test_stream_oracle_cpu.py) and run last, so that `pytest -x` reports as much as possible before a first failure.
VISITED_STREAMS = ("b_", "c1_", "c2_", "c3_", "cip_", "i_", "p_", "wpp_")


def pytest_collection_modifyitems(config, items):
    def late(item):
        if item.get_closest_marker("late"):
            return 1
        stream = getattr(item, "callspec", None) and item.callspec.params.get("stream")
        return int(isinstance(stream, str) and not os.path.basename(stream).startswith(VISITED_STREAMS))
    items.sort(key=late)            # stable: the order inside both groups stays the usual one


@pytest.fixture(scope="session")
def built():
    """build everything that can be built here (CUDA library cross-compiles without a GPU)"""
    import __graft_entry__ as g
    g.build()
    return True
