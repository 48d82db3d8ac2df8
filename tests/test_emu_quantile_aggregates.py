"""Quantile aggregates checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py): tests/test_gpu_quantile_aggregates.py
under thread order 0 with guard pages behind every device allocation, and under a random thread order.  The bitonic sorts of the quantile kernels
exchange keys between lanes (shuffles) and through shared memory between barriers, and the radix passes fill shared histograms that a block
flushes after a barrier: a missing barrier is a wrong quantile under the random order, a read past a group's keys a crash under the guard
pages."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_quantile_aggregates.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_quantile_aggregate_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
