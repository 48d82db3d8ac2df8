"""The fused aggregate's shape checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py):
tests/test_gpu_fused_shape.py under thread order 0 with guard pages behind every device allocation, and under a random order."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_fused_shape.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_fused_shape_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
