"""The GPU parity tests, run WITHOUT a GPU against the emulated build of the library (tests/emu/cuda_emu.h + build_engine_emu.py: the
product's own kernels and host code compiled by g++, every CUDA thread a coroutine, every barrier / warp collective a rendezvous,
cudaMalloc'ed memory filled with 0xCD).  What this adds to the `-m gpu` run on an H100:

* the kernels' LOGIC is checked on every `pytest -m "not gpu"` run, here and on the driver's CPU box;
* threads run in a chosen order between two barriers (HORAE_EMU_ORDER): a missing __syncthreads() / __syncwarp() that the hardware's
  scheduling hides becomes a wrong result or a scheduler error (lanes meeting in different collectives, a collective naming an exited
  lane, a barrier that cannot complete);
* an out-of-bounds access is a segfault with the kernel, block and thread named (with HORAE_EMU_GUARD every allocation, arena
  sub-allocations included, ends at an inaccessible page); uninitialised device memory is 0xCD…, not the zeros a fresh cudaMalloc usually
  returns (that is how the unbounded level-length read of the fused path was found).

The emulated library is test infrastructure: nothing in horaedb_b200/ loads it, and these tests say nothing about speed.  Runs in
subprocesses (pytest + the emu_plugin) so that this process keeps using libhorae_gpu.so for the host-only tests.

The whole GPU suite minus the tests that need a device pointer in torch / NCCL / 100 M rows passes this way (81 of 87; the config-shape
file alone takes 8 minutes): `PYTHONPATH=tests/emu python -m pytest -p emu_plugin tests/test_gpu_*.py -m gpu`.  The CPU suite runs the
quick files."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
QUICK = ["tests/test_gpu_snappy_fused.py", "tests/test_gpu_fused_edges.py", "tests/test_gpu_sst_writer.py", "tests/test_gpu_binary_append.py",
         "tests/test_gpu_zstd.py", "tests/test_gpu_parity.py", "tests/test_gpu_value_domain.py"]


def _run(order, files, extra=(), guard=False, pinned=False):
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_engine_emu
    build_engine_emu.build()                                     # once, here: the xdist workers below only find it up to date
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "tests", "emu") + os.pathsep + env.get("PYTHONPATH", "")
    env["HORAE_EMU_ORDER"] = str(order)
    env["HORAE_EMU_CRASH_REPORT"] = "1"
    if guard:
        env["HORAE_EMU_GUARD"] = "1"
    if pinned:
        env["HORAE_EMU_PINNED"] = "1"
    cmd = [sys.executable, "-m", "pytest", "-p", "emu_plugin", "-n", "4", "-m", "gpu", "-q", "-p", "no:cacheprovider", *extra, *files]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-40:])
    assert r.returncode == 0, tail
    return tail


@pytest.mark.parametrize("order,guard,pinned", [(0, True, False), (2, False, True)])
def test_gpu_parity_tests_on_the_emulated_library(order, guard, pinned):
    # order 0: threads 0..n-1 in turn; 2: a fresh random permutation of the runnable threads in every scheduling pass (1 = descending).
    # guard: every device allocation — every arena sub-allocation too — ends (to 16 bytes) at an inaccessible page
    # pinned: host buffers count as pinned memory, so transient loads take the zero-copy gather kernel instead of one memcpy per range
    tail = _run(order, QUICK, guard=guard, pinned=pinned)
    assert " passed" in tail and "failed" not in tail


def test_damaged_ssts_through_the_emulated_library():
    """tests/emu/fuzz_engine.py: damaged footers, page headers and page bytes (rows that contradict their statistics and their sort order,
    levels / dictionary indices / delta headers / compressed streams that lie) through aggregate (fused and general), scan, compaction
    and the device SST writer — with guard pages behind every device allocation.  Every call returns a result or an error; a crash or a
    kernel that never ends fails the test.  (What a longer run of this tool found is listed in DESIGN.md.)"""
    env = dict(os.environ)
    env["HORAE_EMU_GUARD"] = "1"
    env["HORAE_EMU_CRASH_REPORT"] = "1"
    r = subprocess.run(["timeout", "-s", "SEGV", "600", sys.executable, os.path.join(ROOT, "tests", "emu", "fuzz_engine.py"), "5", "40"],
                       cwd=ROOT, env=env, capture_output=True, text=True)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    last = r.stdout.strip().splitlines()[-1].split()
    assert last[0] == "accepted" and int(last[1]) > 50 and int(last[3]) > 50, tail


def test_random_tables_against_the_oracle_on_the_emulated_library():
    """tests/emu/diff_engine.py: random schemas / NULL rates / key densities / duplicates, 1-4 overlapping files written with random codecs,
    row-group sizes, dictionaries and DELTA_BINARY_PACKED, random predicates and engine flags — scan (batch boundaries, builtin columns),
    aggregate (bit-exact f64 sums) and compaction against the CPU oracle."""
    env = dict(os.environ)
    env["HORAE_EMU_GUARD"] = "1"
    env["HORAE_EMU_CRASH_REPORT"] = "1"
    r = subprocess.run(["timeout", "-s", "SEGV", "900", sys.executable, os.path.join(ROOT, "tests", "emu", "diff_engine.py"), "7", "40"],
                       cwd=ROOT, env=env, capture_output=True, text=True)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0 and "40 cases ok" in r.stdout, tail


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_combine_with_ranks_as_threads(world):
    """tests/emu/combine_check.py: hg_comm_init / hg_agg_combine (csrc/comm.cu: all-gather of per-rank partials, GATHER for disjoint keys,
    REDUCE — sort by key, rank-ordered f64 adds — for keys that cross ranks) with `world` engines of the emulated build in threads and
    tests/emu/nccl_emu.cpp behind comm.cu's dlopen; every rank's result against the oracle's multi-shard definition.  (The same checks run
    on real GPUs in tools/nccl_combine_check.py: world 1 and 2 there, up to 8 here.)"""
    r = subprocess.run(["timeout", "-s", "SEGV", "600", sys.executable, os.path.join(ROOT, "tests", "emu", "combine_check.py"), str(world)],
                       cwd=ROOT, capture_output=True, text=True)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0 and f"world {world}: ok" in r.stdout, tail


def test_plain_c_binding_on_the_emulated_library(tmp_path):
    """tests/c/c_abi_smoke.c — the header bound from plain C, as the Rust FFI would — linked against the emulated build: the full call
    sequence (engine, schema, predicates, aggregate over an Arrow C stream, scan, error paths) runs to "ok" without a GPU."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_engine_emu
    lib = build_engine_emu.build()
    sys.path.insert(0, ROOT)
    from horaedb_b200 import sstgen
    data, _ = sstgen.synth_sst(0, 64, 300, 1000, seq=5, compression="snappy")
    sst = tmp_path / "5.sst"
    sst.write_bytes(data)
    exe = str(tmp_path / "c_abi_smoke_emu")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "c", "c_abi_smoke.c"),
                           "-o", exe, lib, f"-Wl,-rpath,{os.path.dirname(lib)}", "-lstdc++"])
    p = subprocess.run([exe, str(sst)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and "c_abi_smoke: ok" in p.stdout, p.stdout + p.stderr
