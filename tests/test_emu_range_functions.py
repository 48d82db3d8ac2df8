"""Range functions checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py): tests/test_gpu_range_functions.py
under thread order 0 with guard pages behind every device allocation, and under a random thread order.  The function kernel reads back from
a window's end and forward from its start, and the by-map call sorts, cuts and reduces the windows through device counts: a read past a
window or a count a crash under the guard pages, a missing barrier a wrong group under the random order.  The cases the file marks
device_only are deselected here."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_range_functions.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_range_function_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
