"""Range-vector aggregates on the H100: `hg_scan_range_aggregate` and `hg_scan_range_quantile_aggregate` over a PromQL grid.  Prints one
JSON line.

Files: those of tools/bench_counter.py (bench.py's generator: 16 resident SSTs of 6 250 series x 1 000 points, 10 s apart, uncompressed,
100 M rows).  Grid: every 60 s over the data's whole span, with range 60 s, 300 s and 3 600 s (each sample lies in range / step windows).
Per call, the median and [min, max] of `runs` calls after a warm-up, every call returning its Arrow table, and the window count:
  * `range`: hg_scan_range_aggregate (ten columns per window);
  * `range_quantile`: hg_scan_range_quantile_aggregate with q = (0.5, 0.9, 0.99), for range 60 s and 300 s;
  * the k = 1 yardstick: the bucket calls at w = 60 s, hg_scan_aggregate under HG_FLAG_NO_FUSED (the pipeline the range calls run on) and
    hg_scan_counter_aggregate.
gpu_ms is the call's device time (the engine's events, the result's copy to the host included).  `kernels`: each range kernel's time from a
torch.profiler run of its own (one call per range), with the bytes it must move at least and the rate that gives:
  range_gather_kernel      per row: row id 4, time 8, value 8, validity 1 read; time 8, value 8, validity 1 written
  range_count_kernel       per row: time 8, head flag 1 read, count 4 written
  range_offsets_kernel     per row: count 4 read, offset 4 written
  range_windows_kernel     per window: lo 4, hi 4, t 8, key 8 written (its binary searches are not counted)
  reduce_range_windows_kernel  per row once: time 8, value 8, validity 1; per window: lo / hi 8 read, 9 x 8 + 1 written.  Its loops read
                           every row once per window holding it (rows x range / step visits); the minimum counts each row once.
`parity`: with range = step = 60 s and the grid shifted to t = bucket + 59 999 ms (integer times: (t - w, t] = [bucket, bucket + w)), the
range call's count / sum / min / max equal hg_scan_aggregate's and its counter columns hg_scan_counter_aggregate's, bit for bit.
`gpu` names the card and its power limit (nvidia-smi, read only).

Usage: bench_range.py [files=16] [runs=5]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench as shape                                  # noqa: E402  (the benchmark's SST generator)

FILES = int(sys.argv[1]) if len(sys.argv) > 1 else 16
RUNS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
STEP_MS = 60_000
RANGES = (60_000, 300_000, 3_600_000)
QUANTILE_RANGES = (60_000, 300_000)
KERNELS = ("range_gather_kernel", "range_count_kernel", "range_scan_sums_kernel", "range_offsets_kernel", "range_windows_kernel",
           "reduce_range_windows_kernel", "quantile_classify_windows_kernel")


def _spread(xs):
    return {"median": round(float(np.median(xs)), 3), "min": round(float(min(xs)), 3), "max": round(float(max(xs)), 3)}


def _bits(col):
    a = col.combine_chunks().fill_null(0).to_numpy(zero_copy_only=False)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_FLAG_NO_FUSED, Engine, SchemaHandle, SstInput
    shape.SERIES_PER_FILE, shape.POINTS, shape.DELTA_MS = 6250, 1000, 10_000
    files = shape.gen_ssts(0, "none", FILES, min(16, os.cpu_count() or 1))
    if not torch.cuda.is_available():
        sys.exit("bench_range.py needs a GPU")
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
    start = sstgen.T0_MS // STEP_MS * STEP_MS
    end = sstgen.T0_MS + shape.POINTS * shape.DELTA_MS
    qs = (0.5, 0.9, 0.99)

    def timed(flags, fn):
        eng.set_flags(flags)
        t = fn()                                         # warm-up
        gms = []
        for _ in range(RUNS):
            t = fn()
            gms.append(eng.stats()["gpu_ms"])
        st = eng.stats()
        eng.set_flags(0)
        return t, {"gpu_ms": _spread(gms), "windows_or_groups": t.num_rows, "path": st["path"], "kernel_launches": st["kernel_launches"],
                   "bytes_d2h": st["bytes_d2h"]}

    out = {"workload": f"range windows every {STEP_MS // 1000} s: {FILES} resident SSTs, {rows} rows, uncompressed", "gpu": gpu, "rows": rows,
           "runs": RUNS, "grid": {"start_ms": start, "end_ms": end, "step_ms": STEP_MS}}
    kw = dict(group_col=0, ts_col=1, window_ms=STEP_MS, value_col=2)
    _, out["bucket_aggregate_general"] = timed(HG_FLAG_NO_FUSED, lambda: eng.scan_aggregate(handle, ins, [], **kw))
    _, out["bucket_counter"] = timed(0, lambda: eng.scan_counter_aggregate(handle, ins, [], window_ms=STEP_MS))
    windows = {}
    for rng_ in RANGES:
        res = {}
        t, res["range"] = timed(0, lambda: eng.scan_range_aggregate(handle, ins, [], start, end, STEP_MS, rng_))
        windows[rng_] = t.num_rows
        res["windows"] = t.num_rows
        res["row_visits"] = int(sum(t["count"].to_numpy()))
        if rng_ in QUANTILE_RANGES:
            _, res["range_quantile"] = timed(0, lambda: eng.scan_range_quantile_aggregate(handle, ins, [], start, end, STEP_MS, rng_, quantiles=qs))
        out[f"range_{rng_ // 1000}s"] = res

    # parity with the bucket calls: range = step = w, t = bucket + w - 1
    eng.set_flags(HG_FLAG_NO_FUSED)
    rg = eng.scan_range_aggregate(handle, ins, [], start + STEP_MS - 1, end + STEP_MS, STEP_MS, STEP_MS)
    agg = eng.scan_aggregate(handle, ins, [], **kw)
    ctr = eng.scan_counter_aggregate(handle, ins, [], window_ms=STEP_MS)
    eng.set_flags(0)
    parity = rg.num_rows == agg.num_rows == ctr.num_rows
    if parity:
        parity &= bool(np.array_equal(rg["t"].to_numpy() - (STEP_MS - 1), agg["bucket"].to_numpy()))
        parity &= bool(np.array_equal(rg["series_id"].to_numpy(), agg["series_id"].to_numpy()))
        for name in ("count", "sum", "min", "max"):
            parity &= bool(np.array_equal(_bits(rg[name]), _bits(agg[name])))
        for name in ("first_ts", "first_value", "last_ts", "last_value", "increase", "resets"):
            parity &= bool(np.array_equal(_bits(rg[name]), _bits(ctr[name])))
            parity &= rg[name].null_count == ctr[name].null_count
    out["parity"] = bool(parity)

    # kernel times: a profiled run of its own, one call per range (the quantile call at 300 s)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for rng_ in RANGES:
            eng.scan_range_aggregate(handle, ins, [], start, end, STEP_MS, rng_)
        eng.scan_range_quantile_aggregate(handle, ins, [], start, end, STEP_MS, 300_000, quantiles=qs)
        torch.cuda.synchronize()
    times = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k + "(" in ev.key or ev.key.endswith(k):
                times[k] += ev.device_time_total / 1e3        # us -> ms
    n_calls = len(RANGES)
    W = sum(windows.values())
    min_bytes = {"range_gather_kernel": (n_calls + 1) * rows * (4 + 8 + 8 + 1 + 8 + 8 + 1),
                 "range_count_kernel": (n_calls + 1) * rows * (8 + 1 + 4),
                 "range_offsets_kernel": (n_calls + 1) * rows * 8,
                 "range_windows_kernel": (W + windows[300_000]) * 24,
                 "reduce_range_windows_kernel": n_calls * rows * 17 + W * (8 + 9 * 8 + 1)}
    out["kernels"] = {"calls": "3 range calls (60 s, 300 s, 3 600 s) + 1 range quantile call (300 s)"}
    for k in KERNELS:
        e = {"ms": round(times[k], 3)}
        if k in min_bytes:
            e["min_bytes"] = min_bytes[k]
            e["GBps"] = round(min_bytes[k] / (times[k] / 1e3) / 1e9, 1) if times[k] else None
        out["kernels"][k] = e
    print(json.dumps(out))
    eng.close()
    if not parity:
        sys.exit("the range call at range = step differs from the bucket calls")


if __name__ == "__main__":
    main()
