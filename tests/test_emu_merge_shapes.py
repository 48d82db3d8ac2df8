"""The k-way merge and dedup at the limits of their shape checked WITHOUT a GPU on the emulated build of the library (see
test_emu_engine.py): tests/test_gpu_merge_shapes.py under thread order 0 with guard pages behind every device allocation, and under a
random order.  The multi-million-row cases (`*_large`) stay on the GPU; the ~120 000-row range-and-round case runs here, so a wrong
`keep` flag at a round end or a range cut fails on every CPU run."""
import pytest

from test_emu_engine import _run

FILES = ["tests/test_gpu_merge_shapes.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_merge_shape_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, extra=("-k", "not large"), guard=guard)
    assert " passed" in tail and "failed" not in tail
