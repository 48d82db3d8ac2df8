"""Aggregates by label group checked WITHOUT a GPU on the emulated build of the library (see test_emu_engine.py): tests/test_gpu_group_map.py
under thread order 0 with guard pages behind every device allocation, and under a random thread order.  group_map_kernel stages a tile's
slice of the map in shared memory between barriers and searches it: a missing barrier is a wrong group (or an internal error) under the
random order, a read past the map or the row ids a crash under the guard pages.  And tests/emu/combine_by_map_check.py: the REDUCE combine
of by-map partials with 2 and 4 ranks as threads."""
import os
import subprocess
import sys

import pytest

from test_emu_engine import ROOT, _run

FILES = ["tests/test_gpu_group_map.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_group_map_tests_on_the_emulated_library(order, guard):
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail


@pytest.mark.parametrize("world", [2, 4])
def test_reduce_of_by_map_partials_with_ranks_as_threads(world):
    r = subprocess.run(["timeout", "-s", "SEGV", "600", sys.executable, os.path.join(ROOT, "tests", "emu", "combine_by_map_check.py"), str(world)],
                       cwd=ROOT, capture_output=True, text=True)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0 and f"world {world}: ok" in r.stdout, tail
