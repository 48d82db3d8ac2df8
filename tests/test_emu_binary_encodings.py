"""Dictionary-encoded and DELTA_BYTE_ARRAY Binary columns checked WITHOUT a GPU on the emulated build of the library (see
test_emu_engine.py): tests/test_gpu_binary_encodings.py under two thread orders, and damaged SSTs of both encodings through scan and
hg_compact_open (tests/emu/fuzz_binary_encodings.py).  Guard pages turn a read past a dictionary page, a length run
or the DELTA_BYTE_ARRAY value buffer into a crash that names kernel, block and thread; the random order catches a missing barrier in the
warp copy of dba_materialise_kernel."""
import os
import subprocess
import sys

import pytest

from test_emu_engine import ROOT, _run

FILES = ["tests/test_gpu_binary_encodings.py"]


@pytest.mark.parametrize("order,guard", [(0, True), (2, False)])
def test_binary_encoding_tests_on_the_emulated_library(order, guard):
    # order 0: threads in turn, with guard pages behind every device allocation; 2: a fresh random order in every scheduling pass
    tail = _run(order, FILES, guard=guard)
    assert " passed" in tail and "failed" not in tail


@pytest.mark.parametrize("kinds", [["dict", "dict-append"], ["dba", "dba-append"]])
def test_damaged_binary_encodings_end_in_a_result_or_an_error(kinds):
    """Overwritten bytes and flipped bits in dictionary pages, index runs, both length runs and suffix bytes (and the footer): every call
    returns rows or an HgError, and no kernel touches memory outside its buffers."""
    env = dict(os.environ)
    env["HORAE_EMU_GUARD"] = "1"
    env["HORAE_EMU_CRASH_REPORT"] = "1"
    r = subprocess.run(["timeout", "-s", "SEGV", "900", sys.executable, os.path.join(ROOT, "tests", "emu", "fuzz_binary_encodings.py"), "11", "150", *kinds],
                       cwd=ROOT, env=env, capture_output=True, text=True)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    last = r.stdout.strip().splitlines()[-1].split()
    assert last[0] == "accepted" and int(last[1]) > 20 and int(last[3]) > 20, tail
