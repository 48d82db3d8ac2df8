"""Predicates on Binary columns checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py):
tests/test_gpu_binary_predicates.py under thread order 0 with guard pages behind every device allocation, and under a random order.
The byte compares read a row's value and a literal 8 bytes at a time: a read past either ends in a crash that names the kernel, block
and thread, not in a passing test."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_binary_predicates.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_binary_predicate_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
