"""Gate bits of the fused scan checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py):
tests/test_gpu_gate_bits.py under thread order 0 with guard pages behind every device allocation, and under a random order.  The gate job
writes a bitmap behind every row group's decompression regions and the fused kernel reads it two words at a time: a write or read past
the bitmap ends in a crash that names the kernel, block and thread, not in a passing test."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_gate_bits.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_gate_bits_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
