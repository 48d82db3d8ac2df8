"""Pages from other encoders checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py): tests/test_gpu_foreign_pages.py
under thread order 0 with guard pages behind every device allocation, and under a random thread order.  The streams put element
boundaries, copies and frame headers where the page decoders, the gate-bit path and the in-place reads of stored pages have not met them:
a read past a page or a literal is a crash under the guard pages, a missing barrier a wrong row under the random order."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_foreign_pages.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_foreign_pages_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
