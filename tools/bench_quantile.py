"""Quantile aggregates on the H100: `hg_scan_quantile_aggregate` with q = (0.5, 0.9, 0.99).  Prints one JSON line.

Files: those of tools/bench_counter.py (bench.py's generator: 16 resident SSTs of 6 250 series x 1 000 points, 10 s apart, uncompressed,
100 M rows).  Workloads, each the median and [min, max] of `runs` calls after a warm-up, every call returning its Arrow table:
  (a) `series_1min`: per series and 1-minute window (16.7 M groups of 6 rows), beside hg_scan_aggregate under HG_FLAG_NO_FUSED (the
      pipeline the quantile call runs on) and hg_scan_counter_aggregate on the same spec;
  (b) `series`: per series, no window (100 000 groups of 1 000 rows); also today's route without the call: hg_scan_open of the same
      rows to the host, numpy lexsort and a pick per group (host wall clock), and whether its result equals the call's bit for bit;
  (c) `global`: one group of 100 M rows;
  (d) `tag_1min_hash`: HASH per (tag, 1-minute window), beside hg_scan_aggregate under HG_FLAG_NO_FUSED (the same grouping).
gpu_ms is the call's device time (the engine's events, the result's copy to the host included).  `kernels`: each quantile kernel's time
per workload from a torch.profiler run of its own (one call each).  `selection` = the tier kernels (small, medium, hist + resolve) against
the least bytes a selection moves: 8 B per non-NULL value read once and 8 B x Q per group written, as a share of 3.35 TB/s (H100 SXM
HBM3).  The large tier (hist) reads its keys once per radix pass: 8 times.  `gpu` names the card and its power limit (nvidia-smi, read
only).

Usage: bench_quantile.py [files=16] [runs=5]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench as shape                                  # noqa: E402  (the benchmark's SST generator)

FILES = int(sys.argv[1]) if len(sys.argv) > 1 else 16
RUNS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
WINDOW_MS = 60_000
QS = (0.5, 0.9, 0.99)
KERNELS = ("quantile_flags_kernel", "compact_count_kernel", "compact_scan_sums_kernel", "compact_write_kernel", "quantile_keys_kernel",
           "quantile_classify_kernel", "quantile_small_kernel", "quantile_medium_kernel", "quantile_hist_kernel", "quantile_resolve_kernel")
SELECTION = ("quantile_small_kernel", "quantile_medium_kernel", "quantile_hist_kernel", "quantile_resolve_kernel")
HBM_BPS = 3.35e12


def _spread(xs):
    return {"median": round(float(np.median(xs)), 3), "min": round(float(min(xs)), 3), "max": round(float(max(xs)), 3)}


def _timed(eng, fn):
    fn()                                               # warm-up
    gms = []
    for _ in range(RUNS):
        t = fn()
        gms.append(eng.stats()["gpu_ms"])
    st = eng.stats()
    return t, {"gpu_ms": _spread(gms), "groups": t.num_rows, "kernel_launches": st["kernel_launches"], "bytes_d2h": st["bytes_d2h"]}


def _host_route(eng, handle, ins):
    """(b) without the call: every deduplicated row to the host, then a sort and a pick per series"""
    t0 = time.perf_counter()
    tab = eng.scan(handle, ins, [], projection=[0, 2]).read_all()
    t1 = time.perf_counter()
    sid = tab.column(0).to_numpy()
    val = tab.column(1).to_numpy(zero_copy_only=False).astype(np.float64)
    ok = ~np.isnan(val) if tab.column(1).null_count == 0 else tab.column(1).is_valid().to_numpy(zero_copy_only=False)
    bits = val.view(np.uint64)
    key = np.where(bits >> np.uint64(63), ~bits, bits | np.uint64(1 << 63))            # IEEE totalOrder
    order = np.lexsort((key, sid))
    sid, val = sid[order], val[order]
    keys, start, m = np.unique(sid, return_index=True, return_counts=True)
    out = []
    for q in QS:
        rank = q * (m - 1).astype(np.float64)
        lo = np.floor(rank)
        w = rank - lo
        lo = lo.astype(np.int64)
        hi = np.minimum(lo + 1, m - 1)
        a, b = val[start + lo], val[start + hi]
        out.append(np.where(w == 0, a, a * (1 - w) + b * w))
    t2 = time.perf_counter()
    assert ok.all()                                    # the generator writes no NULL and no NaN value
    return keys, out, {"scan_to_host_s": round(t1 - t0, 3), "sort_and_pick_s": round(t2 - t1, 3), "total_s": round(t2 - t0, 3)}


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_AGG_HASH, HG_FLAG_NO_FUSED, Engine, SchemaHandle, SstInput
    shape.SERIES_PER_FILE, shape.POINTS, shape.DELTA_MS = 6250, 1000, 10_000
    if not torch.cuda.is_available():
        sys.exit("bench_quantile.py needs a GPU")
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
    specs = {"series_1min": dict(group_col=0, ts_col=1, window_ms=WINDOW_MS, value_col=2),
             "series": dict(group_col=0, ts_col=1, window_ms=0, value_col=2),
             "global": dict(group_col=-1, ts_col=1, window_ms=0, value_col=2),
             "tag_1min_hash": dict(group_col=3, ts_col=1, window_ms=WINDOW_MS, value_col=2, mode=HG_AGG_HASH)}
    out = {"workload": f"quantiles q={list(QS)}: {FILES} resident SSTs, {rows} rows, uncompressed", "gpu": gpu, "rows": rows, "runs": RUNS}
    tables = {}
    for name, kw in specs.items():
        eng.set_flags(0)
        tables[name], res = _timed(eng, lambda: eng.scan_quantile_aggregate(handle, ins, [], quantiles=QS, **kw))
        out[name] = {"quantile": res}
    eng.set_flags(HG_FLAG_NO_FUSED)
    _, out["series_1min"]["aggregate_general"] = _timed(eng, lambda: eng.scan_aggregate(handle, ins, [], **specs["series_1min"]))
    _, out["tag_1min_hash"]["aggregate_general"] = _timed(eng, lambda: eng.scan_aggregate(handle, ins, [], **specs["tag_1min_hash"]))
    eng.set_flags(0)
    _, out["series_1min"]["counter"] = _timed(eng, lambda: eng.scan_counter_aggregate(handle, ins, [], **specs["series_1min"]))
    a = out["series_1min"]
    a["quantile_over_counter"] = round(a["quantile"]["gpu_ms"]["median"] / a["counter"]["gpu_ms"]["median"], 3)
    a["quantile_over_general"] = round(a["quantile"]["gpu_ms"]["median"] / a["aggregate_general"]["gpu_ms"]["median"], 3)
    # (b) today's route, and its result against the call's
    keys, host_q, host_t = _host_route(eng, handle, ins)
    got = tables["series"]
    same = got.column(0).to_numpy().tolist() == keys.tolist()
    for j in range(len(QS)):
        same &= np.array_equal(got.column(2 + j).to_numpy().view(np.uint64), host_q[j].view(np.uint64))
    out["series"]["host_route"] = dict(host_t, equal_to_call=bool(same))
    # kernel times: a profiled run of its own, one call per workload
    for name, kw in specs.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.scan_quantile_aggregate(handle, ins, [], quantiles=QS, **kw)
            torch.cuda.synchronize()
        times = {k: 0.0 for k in KERNELS}
        for ev in prof.key_averages():
            for k in KERNELS:
                if k + "(" in ev.key or ev.key.endswith(k):
                    times[k] += ev.device_time_total / 1e3     # us -> ms
        groups = tables[name].num_rows
        sel_ms = sum(times[k] for k in SELECTION)
        min_bytes = rows * 8 + groups * 8 * len(QS)            # no NULL values in these files: every row is a value
        out[name]["kernels_ms"] = {k: round(v, 3) for k, v in times.items() if v}
        out[name]["selection"] = {"ms": round(sel_ms, 3), "min_bytes": min_bytes,
                                  "share_of_3.35TBps": round(min_bytes / (sel_ms / 1e3) / HBM_BPS, 3) if sel_ms else None}
    print(json.dumps(out))
    eng.close()
    if not same:
        sys.exit("the host route and the call disagree on (b)")


if __name__ == "__main__":
    main()
