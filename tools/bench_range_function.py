"""`sum by (job) (rate(x[r]))` every 60 s on the H100: today's host route against `hg_scan_range_function` and
`hg_scan_range_function_by_map`.  Prints one JSON line.

Files and grid: those of tools/bench_range.py (16 resident SSTs of 6 250 series x 1 000 points, 10 s apart, uncompressed, 100 M rows; every
60 s over the data's whole span), range 60 s, 300 s and 3 600 s.  Label groups: series_id % G.  Per route, the median and [min, max] of
`runs` calls after a warm-up, each returning its table:
  (a) host:     hg_scan_range_aggregate (ten partial columns per window), then Prometheus's extrapolation of rate and the group sum in
                numpy on the host (G = 100);
  (b) function: hg_scan_range_function(HG_FN_RATE), one value per series and step;
  (c) by_map:   hg_scan_range_function_by_map(HG_FN_RATE) with G = 100 and G = 10 000, one row per group and step.
gpu_ms is the call's device time (the engine's events, the result's copy to the host included); wall_ms the host's time for the whole
route (for (a) with its numpy part).  `parity`: (c)'s count and sum equal (b)'s values counted and summed per (group, t) on the host in
series order, bit for bit.  `gpu` names the card and its power limit (nvidia-smi, read only).

Usage: bench_range_function.py [files=16] [runs=5]"""
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
STEP_MS = 60_000
RANGES = (60_000, 300_000, 3_600_000)
GROUPS = (100, 10_000)


def _spread(xs):
    return {"median": round(float(np.median(xs)), 3), "min": round(float(min(xs)), 3), "max": round(float(max(xs)), 3)}


def host_rate_by_group(t, start, range_ms, G):
    """Prometheus's extrapolatedRate from the range aggregate's columns, then the sum per (series % G, t): the route without the new calls"""
    first_ts = t["first_ts"].to_numpy(zero_copy_only=False)
    last_ts = t["last_ts"].to_numpy(zero_copy_only=False)
    v0 = t["first_value"].to_numpy(zero_copy_only=False)
    result = t["increase"].to_numpy()
    m = t["count"].to_numpy().astype(np.float64)
    tt = t["t"].to_numpy()
    ok = (m >= 2) & (last_ts != first_ts)
    d_start = (first_ts - (tt - range_ms)).astype(np.float64) / 1000
    d_end = (tt - last_ts).astype(np.float64) / 1000
    sampled = (last_ts - first_ts).astype(np.float64) / 1000
    with np.errstate(divide="ignore", invalid="ignore"):
        avg = sampled / (m - 1)
        thr = avg * 1.1
        d_start = np.where(d_start >= thr, avg / 2, d_start)
        d_zero = sampled * (v0 / result)
        d_start = np.where((result > 0) & (v0 >= 0) & (d_zero < d_start), d_zero, d_start)
        d_end = np.where(d_end >= thr, avg / 2, d_end)
        value = result * ((sampled + d_start + d_end) / sampled / (range_ms / 1000))
    key = (t["series_id"].to_numpy() % G) * (1 << 24) + (tt - start) // STEP_MS
    key, value = key[ok], value[ok]
    uniq, inv = np.unique(key, return_inverse=True)
    return uniq, np.bincount(inv, weights=value, minlength=len(uniq))


def main():
    import torch

    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_FN_RATE, Engine, SchemaHandle, SstInput
    shape.SERIES_PER_FILE, shape.POINTS, shape.DELTA_MS = 6250, 1000, 10_000
    files = shape.gen_ssts(0, "none", FILES, min(16, os.cpu_count() or 1))
    if not torch.cuda.is_available():
        sys.exit("bench_range_function.py needs a GPU")
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

    def timed(fn):
        fn()                                             # warm-up
        gms, wall = [], []
        for _ in range(RUNS):
            t0 = time.perf_counter()
            t = fn()
            wall.append((time.perf_counter() - t0) * 1e3)
            gms.append(eng.stats()["gpu_ms"])
        st = eng.stats()
        return t, {"gpu_ms": _spread(gms), "wall_ms": _spread(wall), "bytes_d2h": st["bytes_d2h"], "rows_out": int(st["groups_out"])}

    out = {"workload": f"sum by (series % G) (rate(x[range])) every {STEP_MS // 1000} s: {FILES} resident SSTs, {rows} rows, uncompressed",
           "gpu": gpu, "rows": rows, "runs": RUNS, "grid": {"start_ms": start, "end_ms": end, "step_ms": STEP_MS}}
    parity = True
    for rng_ in RANGES:
        res = {}

        def host_route():
            t = eng.scan_range_aggregate(handle, ins, [], start, end, STEP_MS, rng_)
            host_route.windows = t.num_rows
            return host_rate_by_group(t, start, rng_, GROUPS[0])
        (keys_a, _), res["a_host_g100"] = timed(host_route)
        res["a_host_g100"]["windows"] = host_route.windows
        res["a_host_g100"]["rows_out"] = len(keys_a)
        per, res["b_function"] = timed(lambda: eng.scan_range_function(handle, ins, HG_FN_RATE, [], start, end, STEP_MS, rng_))
        sid = per["series_id"].to_numpy()
        series = np.unique(sid)
        for G in GROUPS:
            groups = (series % G).astype(np.uint32)
            got, res[f"c_by_map_g{G}"] = timed(lambda: eng.scan_range_function_by_map(handle, ins, HG_FN_RATE, series, groups, [], start, end,
                                                                                       STEP_MS, rng_))
            # (b) summed per (group, t) in series order: bincount adds its weights in input order, (b) is in (series, t) order
            key = (sid % G).astype(np.int64) * (1 << 24) + (per["t"].to_numpy() - start) // STEP_MS
            uniq, inv = np.unique(key, return_inverse=True)
            sums = np.bincount(inv, weights=per["value"].to_numpy(), minlength=len(uniq))
            counts = np.bincount(inv, minlength=len(uniq))
            gkey = got["group"].to_numpy().astype(np.int64) * (1 << 24) + (got["t"].to_numpy() - start) // STEP_MS
            ok = len(gkey) == len(uniq) and bool(np.array_equal(gkey, uniq))
            ok = ok and bool(np.array_equal(got["count"].to_numpy(), counts.astype(np.uint64)))
            ok = ok and bool(np.array_equal(got["sum"].to_numpy().view(np.uint64), sums.view(np.uint64)))
            res[f"c_by_map_g{G}"]["parity"] = ok
            parity &= ok
        out[f"range_{rng_ // 1000}s"] = res
    out["parity"] = bool(parity)
    print(json.dumps(out))
    eng.close()
    if not parity:
        sys.exit("the by-map call differs from the per-series values summed on the host")


if __name__ == "__main__":
    main()
