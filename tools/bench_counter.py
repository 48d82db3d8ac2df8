"""Counter aggregates on the H100: `hg_scan_counter_aggregate` next to `hg_scan_aggregate` on the same query.  Prints one JSON line.

Shape: config 3 of tools/bench_downsample.py (bench.py's generator: 16 resident SSTs of 6 250 series x 1 000 points, 10 s apart,
uncompressed), 1-minute windows, no predicate; plus one run with `series_id IN_SET (1 000 series) AND ts in [a, b)`.  Per query, the
median and [min, max] of `runs` calls after a warm-up, every call returning its Arrow table:
  * `aggregate_fused`: hg_scan_aggregate as a caller runs it (the fused scan where it applies);
  * `aggregate_general`: hg_scan_aggregate with HG_FLAG_NO_FUSED, the pipeline the counter call runs on;
  * `counter`: hg_scan_counter_aggregate.
gpu_ms is the call's device time (the engine's events, the result's copy to the host included).  `reduce` gives
reduce_counter_groups_kernel's and reduce_groups_kernel's time from a torch.profiler run of its own (one call each, no predicate), with
the bytes each must move at least: per row the 4-byte row id and the 8-byte value; per group the segment start, the key and the first
row's time (read) and the outputs (written: 6 x 8 bytes for reduce_groups, 8 x 8 + 1 for the counter kernel, which also reads the last
valid row's time).  `gpu` names the card and its power limit (nvidia-smi, read only).

Usage: bench_counter.py [files=16] [runs=5]"""
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
WINDOW_MS = 60_000
KERNELS = ("reduce_counter_groups_kernel", "reduce_groups_kernel")


def _spread(xs):
    return {"median": round(float(np.median(xs)), 3), "min": round(float(min(xs)), 3), "max": round(float(max(xs)), 3)}


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_FLAG_NO_FUSED, Engine, SchemaHandle, SstInput
    shape.SERIES_PER_FILE, shape.POINTS, shape.DELTA_MS = 6250, 1000, 10_000
    files = shape.gen_ssts(0, "none", FILES, min(16, os.cpu_count() or 1))
    if not torch.cuda.is_available():
        sys.exit("bench_counter.py needs a GPU")
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
    kw = dict(group_col=0, ts_col=1, window_ms=WINDOW_MS, value_col=2)
    calls = {
        "aggregate_fused": (0, lambda p: eng.scan_aggregate(handle, ins, p, **kw)),
        "aggregate_general": (HG_FLAG_NO_FUSED, lambda p: eng.scan_aggregate(handle, ins, p, **kw)),
        "counter": (0, lambda p: eng.scan_counter_aggregate(handle, ins, p, **kw)),
    }
    span = shape.POINTS * shape.DELTA_MS
    rng = np.random.default_rng(7)
    ids = rng.choice(FILES * shape.SERIES_PER_FILE, 1000, replace=False).astype(np.uint64)
    queries = {"no_predicate": [],
               "in_set_1000_and_ts_range": [("series_id", "in_set", ids), ("ts", "ge", sstgen.T0_MS + span // 4),
                                            ("ts", "lt", sstgen.T0_MS + 3 * span // 4)]}
    out = {"workload": f"1-min counter partials vs sum/min/max/count: {FILES} resident SSTs, {rows} rows, uncompressed", "gpu": gpu,
           "rows": rows, "runs": RUNS}
    ok = True
    for qname, preds in queries.items():
        res = {}
        for cname, (flags, fn) in calls.items():
            eng.set_flags(flags)
            t = fn(preds)                                # warm-up
            gms = []
            for _ in range(RUNS):
                t = fn(preds)
                gms.append(eng.stats()["gpu_ms"])
            st = eng.stats()
            res[cname] = {"gpu_ms": _spread(gms), "groups": t.num_rows, "path": st["path"], "kernel_launches": st["kernel_launches"],
                          "bytes_d2h": st["bytes_d2h"]}
        eng.set_flags(0)
        groups = {v["groups"] for v in res.values()}
        ok &= len(groups) == 1
        res["counter_over_general"] = round(res["counter"]["gpu_ms"]["median"] / res["aggregate_general"]["gpu_ms"]["median"], 3)
        out[qname] = res
    # kernel times: a profiled run of its own, one call of each general-pipeline reducer
    groups = out["no_predicate"]["counter"]["groups"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.set_flags(HG_FLAG_NO_FUSED)
        eng.scan_aggregate(handle, ins, [], **kw)
        eng.set_flags(0)
        eng.scan_counter_aggregate(handle, ins, [], **kw)
        torch.cuda.synchronize()
    times = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k + "(" in ev.key or ev.key.endswith(k):
                times[k] += ev.device_time_total / 1e3        # us -> ms
    min_bytes = {"reduce_counter_groups_kernel": rows * 12 + groups * (4 + 8 + 8 + 8 + 8 * 8 + 1),
                 "reduce_groups_kernel": rows * 12 + groups * (4 + 8 + 8 + 6 * 8)}
    out["reduce"] = {k: {"ms": round(times[k], 3), "min_bytes": min_bytes[k],
                         "GBps": round(min_bytes[k] / (times[k] / 1e3) / 1e9, 1) if times[k] else None} for k in KERNELS}
    out["parity_groups"] = ok
    print(json.dumps(out))
    eng.close()
    if not ok:
        sys.exit("the three calls returned different group counts")


if __name__ == "__main__":
    main()
