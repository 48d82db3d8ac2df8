"""Top-k per label group checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py): tests/test_gpu_range_topk.py
under thread order 0 with guard pages behind every device allocation, and under a random thread order.  The call sorts the windows twice,
cuts them into (group, t) segments, searches each window's segment and gathers the kept ones through device counts: a read past a segment
or a count is a crash under the guard pages, a missing barrier a wrong row under the random order.  The cases the file marks device_only
are deselected here."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_range_topk.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_range_topk_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
