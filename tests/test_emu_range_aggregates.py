"""Range aggregates checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py): tests/test_gpu_range_aggregates.py
under thread order 0 with guard pages behind every device allocation, and under a random thread order.  The window enumeration scans block
sums across blocks and binary-searches the per-row offsets, and overlapping windows point into one key array of the quantile tiers: a
missing barrier is a wrong window under the random order, a read past a window's rows or keys a crash under the guard pages.  The cases
the file marks device_only are deselected here."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_range_aggregates.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_range_aggregate_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
