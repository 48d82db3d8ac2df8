"""Pages laid out by other writers checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py):
tests/test_gpu_foreign_encodings.py under thread order 0 with guard pages behind every device allocation, and under a random thread
order.  The layouts put DELTA miniblocks, bit-packed runs and level runs where the decoders have not met them: a read past a page or a
miniblock is a crash under the guard pages, a missing barrier a wrong row under the random order."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_foreign_encodings.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_foreign_encodings_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
