"""Bloom filters of the GPU SST writer and the scan planner, checked WITHOUT a GPU on the emulated build of the library (see
test_emu_engine.py): tests/test_gpu_bloom_filters.py under two thread orders.  The pinned SHA-256 of its output must hold under both, so
the bitsets — built with atomicOr in shared or global memory — do not depend on the order threads run in."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_bloom_filters.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_bloom_filter_tests_on_the_emulated_library(order, guard):
    # order 0: threads in turn, with guard pages behind every device allocation; 2: a fresh random order in every scheduling pass
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
