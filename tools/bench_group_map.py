"""Aggregates by label group on the H100 (`hg_scan_aggregate_by_map`, `hg_scan_quantile_aggregate_by_map`).  Prints one JSON line.

Files: those of tools/bench_quantile.py (bench.py's generator: 16 resident SSTs of 6 250 series x 1 000 points, 10 s apart,
uncompressed, 100 M rows of 100 000 series).  Workloads, each the median and [min, max] of `runs` calls after a warm-up, every call
returning its Arrow table:
  (a) `map_G`: every series mapped into G = 1 / 16 / 1 000 / 100 000 groups (ordinal = series mod G), per 1-minute window.  Beside them
      `hash_tag_1min`: hg_scan_aggregate HASH on (tag, window) under HG_FLAG_NO_FUSED, the same grouping work without the lookup; and
      `host_route`: today's route, per-series partials per window to the host (hg_scan_aggregate) and a numpy group reduce for G = 1 000
      (host wall clock), with the largest relative difference of its sums from the call's;
  (b) `map_1000_series`: a map of 1 000 series into 16 groups, with and without HG_FLAG_NO_PRUNING: rows_decoded and gpu_ms;
  (c) `quantiles_16`: q = (0.5, 0.9, 0.99) by a 16-group map per 1-minute window;
  (d) `group_map_kernel`: its time in a torch.profiler run of its own (the G = 1 000 call) against the bytes it must move at least, 12 B
      read (row id + 8-byte key) and 4 B written per row, as a share of 3.35 TB/s (H100 SXM HBM3);
  (e) `planning`: the host's map preparation for 16 777 216 keys, sorted and shuffled, from the library's HORAE_TRACE line.
gpu_ms is the call's device time (the engine's events, the result's copy to the host included).  `gpu` names the card and its power
limit (nvidia-smi, read only).

Usage: bench_group_map.py [files=16] [runs=5]"""
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["HORAE_TRACE"] = "1"                       # read once by the library: its planning lines go to stderr, captured below
import bench as shape                                  # noqa: E402  (the benchmark's SST generator)

FILES = int(sys.argv[1]) if len(sys.argv) > 1 else 16
RUNS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
WINDOW_MS = 60_000
QS = (0.5, 0.9, 0.99)
HBM_BPS = 3.35e12


class _Stderr:
    """fd 2 into a temporary file (the library writes its trace there), text in .text"""
    def __enter__(self):
        sys.stderr.flush()
        self.tmp = tempfile.TemporaryFile()
        self.saved = os.dup(2)
        os.dup2(self.tmp.fileno(), 2)
        return self

    def __exit__(self, *a):
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.tmp.seek(0)
        self.text = self.tmp.read().decode(errors="replace")
        self.tmp.close()


def _spread(xs):
    return {"median": round(float(np.median(xs)), 3), "min": round(float(min(xs)), 3), "max": round(float(max(xs)), 3)}


def _timed(eng, fn):
    with _Stderr():
        fn()                                           # warm-up
        gms = []
        for _ in range(RUNS):
            t = fn()
            gms.append(eng.stats()["gpu_ms"])
    st = eng.stats()
    return t, {"gpu_ms": _spread(gms), "groups": t.num_rows, "rows_decoded": st["rows_decoded"], "kernel_launches": st["kernel_launches"]}


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_AGG_HASH, HG_FLAG_NO_FUSED, HG_FLAG_NO_PRUNING, Engine, SchemaHandle, SstInput
    shape.SERIES_PER_FILE, shape.POINTS, shape.DELTA_MS = 6250, 1000, 10_000
    if not torch.cuda.is_available():
        sys.exit("bench_group_map.py needs a GPU")
    files = shape.gen_ssts(0, "none", FILES, min(16, os.cpu_count() or 1))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    ins = []
    for seq, data, n in files:
        eng.load_sst(handle, SstInput(id=seq, data=data))
        ins.append(SstInput(id=seq, num_rows=n))
    rows = sum(n for _, _, n in files)
    n_series = FILES * shape.SERIES_PER_FILE
    sids = np.arange(n_series, dtype=np.uint64)
    spec = dict(group_col=0, ts_col=1, window_ms=WINDOW_MS, value_col=2)
    out = {"workload": f"aggregates by map: {FILES} resident SSTs, {rows} rows, {n_series} series, uncompressed", "gpu": gpu, "rows": rows,
           "runs": RUNS}
    # (a)
    tables = {}
    for G in (1, 16, 1000, 100_000):
        groups = (sids % G).astype(np.uint32)
        tables[G], out[f"map_{G}"] = _timed(eng, lambda: eng.scan_aggregate_by_map(handle, ins, sids, groups, **spec))
    eng.set_flags(HG_FLAG_NO_FUSED)
    _, out["hash_tag_1min"] = _timed(eng, lambda: eng.scan_aggregate(handle, ins, [], group_col=3, ts_col=1, window_ms=WINDOW_MS, value_col=2,
                                                                     mode=HG_AGG_HASH))
    eng.set_flags(0)
    base = out["hash_tag_1min"]["gpu_ms"]["median"]
    out["map_over_hash"] = {f"map_{G}": round(out[f"map_{G}"]["gpu_ms"]["median"] / base, 3) for G in (1, 16, 1000, 100_000)}
    walls = []
    for _ in range(RUNS):
        t0 = time.perf_counter()
        part = eng.scan_aggregate(handle, ins, [], **spec)
        t1 = time.perf_counter()
        g = (part["series_id"].to_numpy() % 1000).astype(np.int64)
        b = part["bucket"].to_numpy()
        key = g * (1 << 40) + (b - b.min()) // WINDOW_MS
        uk, inv = np.unique(key, return_inverse=True)
        sums = np.zeros(len(uk))
        np.add.at(sums, inv, part["sum"].to_numpy())
        t2 = time.perf_counter()
        walls.append((t1 - t0, t2 - t1, t2 - t0))
    got = tables[1000]["sum"].to_numpy()
    rel = float(np.max(np.abs(sums - got) / np.maximum(np.abs(got), 1e-300))) if len(got) == len(sums) else None
    out["host_route"] = {"partials_to_host_s": _spread([w[0] for w in walls]), "numpy_reduce_s": _spread([w[1] for w in walls]),
                         "total_s": _spread([w[2] for w in walls]), "partial_rows": part.num_rows,
                         "max_rel_diff_of_sums": rel}
    # (b)
    rng = np.random.default_rng(1)
    few = np.sort(rng.choice(sids, 1000, replace=False))
    few_groups = (few % 16).astype(np.uint32)
    _, out["map_1000_series"] = _timed(eng, lambda: eng.scan_aggregate_by_map(handle, ins, few, few_groups, **spec))
    eng.set_flags(HG_FLAG_NO_PRUNING)
    _, out["map_1000_series_no_pruning"] = _timed(eng, lambda: eng.scan_aggregate_by_map(handle, ins, few, few_groups, **spec))
    eng.set_flags(0)
    # (c)
    g16 = (sids % 16).astype(np.uint32)
    _, out["quantiles_16"] = _timed(eng, lambda: eng.scan_quantile_aggregate_by_map(handle, ins, sids, g16, quantiles=QS, **spec))
    # (d)
    g1000 = (sids % 1000).astype(np.uint32)
    with _Stderr():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.scan_aggregate_by_map(handle, ins, sids, g1000, **spec)
            torch.cuda.synchronize()
    st = eng.stats()
    kms = sum(ev.device_time_total for ev in prof.key_averages() if "group_map_kernel" in ev.key) / 1e3
    min_bytes = st["rows_out"] * 16
    out["group_map_kernel"] = {"ms": round(kms, 3), "rows": st["rows_out"], "min_bytes": min_bytes,
                               "share_of_3.35TBps": round(min_bytes / (kms / 1e3) / HBM_BPS, 3) if kms else None}
    # (e)
    n = 1 << 24
    big = np.arange(n, dtype=np.uint64) * 7
    big_groups = (big % 1000).astype(np.uint32)
    shuffled = rng.permutation(n)
    plan = {}
    for name, (k, g) in (("sorted", (big, big_groups)), ("unsorted", (big[shuffled], big_groups[shuffled]))):
        with _Stderr() as cap:
            eng.scan_aggregate_by_map(handle, ins[:1], k, g, **spec)
        m = re.findall(r"\[group_map\] (\d+) keys -> (\d+), ([a-z ]+), (\d+) us", cap.text)
        plan[name] = {"keys": int(m[-1][0]), "how": m[-1][2], "host_us": int(m[-1][3])} if m else None
    out["planning"] = plan
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
