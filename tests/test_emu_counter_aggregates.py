"""Counter aggregates checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py): tests/test_gpu_counter_aggregates.py
under thread order 0 with guard pages behind every device allocation, and under a random thread order.  reduce_counter_groups_kernel reads
its group's rows through the `rows` indirection up to the next group's start: a read past a group's last row or past the result's end is a
crash that names the kernel, block and thread under the guard pages."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_counter_aggregates.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_counter_aggregate_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail
