"""Set-membership predicates checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py):
tests/test_gpu_in_set.py under thread order 0 with guard pages behind every device allocation, and under a random order.
eval_in_set_kernel shares one staging buffer between the predicates and the tiles of a block: a missing barrier there is a wrong result
under the random order, and a search that leaves the set's device copy is a crash that names the kernel, block and thread.  The 2^20-value
case is left to the GPU run (its file and set sizes cost the emulation minutes)."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_in_set.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_in_set_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, extra=("-k", "not million"), guard=guard)
    assert " passed" in tail and "failed" not in tail
