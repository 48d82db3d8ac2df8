"""`histogram_quantile(q, sum by (job, le) (rate(x[r])))` every 60 s on the H100: today's route (the by-map range function call with one
ordinal per (group, bound), then Prometheus's bucketQuantile on the host) against `hg_scan_histogram_quantile`.  Prints one JSON line.

Files and grid: those of tools/bench_range.py (16 resident SSTs of 6 250 series x 1 000 points, 10 s apart, uncompressed, 100 M rows; every
60 s over the data's whole span), range 300 s, 60 s and 3 600 s.  Map: series s is the bucket of bound B[s % 12] (11 finite bounds and +inf)
of group (s // 12) % G, G = 100 and 1 000; q = 0.5, 0.9, 0.99; HG_FN_RATE.  Per route, the median and [min, max] of `runs` calls after a
warm-up, each returning its result:
  (a) by_map_host: hg_scan_range_function_by_map with the pair ordinal g * 12 + b, then bucketQuantile vectorised in numpy on the host;
  (b) histogram:   hg_scan_histogram_quantile, one row per (group, t).
gpu_ms is the call's device time (the engine's events, the result's copy to the host included); wall_ms the host's time for the whole route
(for (a) with its numpy part).  `parity`: (b)'s group, t, forced_monotonic and quantiles equal (a)'s, every f64 bit for bit.  `kernels_us`:
the device time per call of the new kernels under torch.profiler, in a separate run.  `gpu` names the card and its power limit
(nvidia-smi, read only).

Usage: bench_histogram_quantile.py [files=16] [runs=5]"""
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
RANGES = (300_000, 60_000, 3_600_000)
GROUPS = (100, 1_000)
BOUNDS = np.array([0.005, 0.01, 0.025, 0.05, 0.1, 0.25, 0.5, 1.0, 2.5, 5.0, 10.0, np.inf])
QS = (0.5, 0.9, 0.99)
MIN_NORMAL = 2.0 ** -1022
MAX_F64 = np.finfo(np.float64).max


def _spread(xs):
    return {"median": round(float(np.median(xs)), 3), "min": round(float(min(xs)), 3), "max": round(float(max(xs)), 3)}


def _almost_equal(a, b):
    """util/almost.Equal(a, b, 1e-12), elementwise"""
    s = np.abs(a) + np.abs(b)
    d = np.abs(a - b)
    tiny = (a == 0) | (b == 0) | (s < MIN_NORMAL)
    m = np.where(np.isnan(s) | (s < MAX_F64), s, MAX_F64)
    rel = d / np.where(tiny, 1.0, m) < 1e-12
    return (np.isnan(a) & np.isnan(b)) | (a == b) | np.where(tiny, d < 1e-12 * MIN_NORMAL, rel)


def bucket_quantile_dense(c, u, qs):
    """include/horae_gpu.h's definition over R rows of n buckets each, all present, bounds u ascending with u[-1] = +inf: (forced, [R] per
    q).  Every operation is one elementwise f64 operation, as in the definition."""
    R, n = c.shape
    c = c.copy()
    prev = c[:, 0].copy()
    forced = np.zeros(R, bool)
    for i in range(1, n):
        cur = c[:, i]
        eq = cur == prev
        ae = ~eq & _almost_equal(prev, cur)
        lt = ~eq & ~ae & (cur < prev)
        c[:, i] = np.where(ae | lt, prev, cur)
        forced |= lt
        prev = np.where(eq | ae | lt, prev, cur)
    obs = c[:, n - 1]
    out = []
    rows = np.arange(R)
    for q in qs:
        rank = q * obs
        lo, hi = np.zeros(R, np.int64), np.full(R, n - 1, np.int64)
        while True:
            act = lo < hi
            if not act.any():
                break
            h = (lo + hi) // 2
            up = ~(c[rows, h] >= rank)
            lo = np.where(act & up, h + 1, lo)
            hi = np.where(act & ~up, h, hi)
        b = lo
        bm = np.maximum(b - 1, 0)
        start = np.where(b > 0, u[bm], 0.0)
        sub = np.where(b > 0, c[rows, bm], 0.0)
        end = u[np.minimum(b, n - 1)]
        with np.errstate(all="ignore"):
            r = start + (end - start) * ((rank - sub) / (c[rows, np.minimum(b, n - 1)] - sub))
        r = np.where((b == 0) & (u[0] <= 0), u[0], r)
        r = np.where(b == n - 1, u[n - 2], r)
        r = np.where(obs == 0, np.nan, r)
        out.append(r)
    return forced, out


def host_route(t, G, start):
    """the by-map rows (pair ordinal g * 12 + b, t, sum) of every (g, t) with all 12 buckets -> the (b) result's columns"""
    nb = len(BOUNDS)
    pair = t["group"].to_numpy().astype(np.int64)
    tt = t["t"].to_numpy()
    sums = t["sum"].to_numpy()
    gt = (pair // nb) * (1 << 24) + (tt - start) // STEP_MS
    uniq, first, cnt = np.unique(gt, return_index=True, return_counts=True)
    if not (cnt == nb).all():
        raise SystemExit("bench_histogram_quantile.py: a (group, t) without all of its buckets")
    # the by-map rows are in (pair, t) order; a (g, t)'s buckets are rows of one g with the same t, one per bound
    order = np.lexsort((pair % nb, gt))
    c = sums[order].reshape(-1, nb)
    forced, qv = bucket_quantile_dense(c, BOUNDS, QS)
    return (uniq >> 24).astype(np.uint32), tt[order][::nb], forced.astype(np.uint8), qv


def main():
    import torch

    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_FN_RATE, Engine, SchemaHandle, SstInput
    shape.SERIES_PER_FILE, shape.POINTS, shape.DELTA_MS = 6250, 1000, 10_000
    files = shape.gen_ssts(0, "none", FILES, min(16, os.cpu_count() or 1))
    if not torch.cuda.is_available():
        sys.exit("bench_histogram_quantile.py needs a GPU")
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
    series = np.arange(FILES * shape.SERIES_PER_FILE, dtype=np.uint64)
    nb = len(BOUNDS)
    bidx = (series % nb).astype(np.int64)
    ubs = BOUNDS[bidx]

    def timed(fn):
        fn()                                             # warm-up
        gms, wall = [], []
        for _ in range(RUNS):
            t0 = time.perf_counter()
            t = fn()
            wall.append((time.perf_counter() - t0) * 1e3)
            gms.append(eng.stats()["gpu_ms"])
        st = eng.stats()
        return t, {"gpu_ms": _spread(gms), "wall_ms": _spread(wall), "bytes_d2h": st["bytes_d2h"], "rows_out": int(st["groups_out"]),
                   "launches": int(st["kernel_launches"])}

    out = {"workload": f"histogram_quantile(q, sum by (g, le) (rate(x[range]))) every {STEP_MS // 1000} s: {FILES} resident SSTs, {rows} rows, "
                       f"uncompressed, {nb} buckets per histogram",
           "gpu": gpu, "rows": rows, "runs": RUNS, "quantiles": QS, "grid": {"start_ms": start, "end_ms": end, "step_ms": STEP_MS}}
    parity = True
    for rng_ in RANGES:
        res = {}
        for G in GROUPS:
            groups = ((series // nb) % G).astype(np.uint32)
            pair_ord = (groups.astype(np.int64) * nb + bidx).astype(np.uint32)

            def route_a():
                t = eng.scan_range_function_by_map(handle, ins, HG_FN_RATE, series, pair_ord, [], start, end, STEP_MS, rng_)
                route_a.stats = eng.stats()
                return host_route(t, G, start)

            def route_b():
                return eng.scan_histogram_quantile(handle, ins, HG_FN_RATE, series, groups, ubs, QS, [], start, end, STEP_MS, rng_)

            a, res[f"a_by_map_host_g{G}"] = timed(route_a)
            st = route_a.stats                               # the device call's own numbers, not the numpy part's
            res[f"a_by_map_host_g{G}"].update({"gpu_ms_last": round(st["gpu_ms"], 3), "bytes_d2h": st["bytes_d2h"], "rows_out": int(st["groups_out"]),
                                               "launches": int(st["kernel_launches"])})
            b, res[f"b_histogram_g{G}"] = timed(route_b)
            ok = b.num_rows == len(a[0]) and b["group"].to_numpy().tolist() == a[0].tolist() and bool(np.array_equal(b["t"].to_numpy(), a[1]))
            ok = ok and bool(np.array_equal(b["forced_monotonic"].to_numpy(), a[2]))
            for j in range(len(QS)):
                x, y = b[f"quantile_{j}"].to_numpy(), a[3][j]
                ok = ok and bool(np.array_equal(np.isnan(x), np.isnan(y)) and np.array_equal(x[~np.isnan(x)].view(np.uint64), y[~np.isnan(y)].view(np.uint64)))
            res[f"b_histogram_g{G}"]["parity"] = ok
            res[f"b_histogram_g{G}"]["forced_rows"] = int(b["forced_monotonic"].to_numpy().sum())
            parity &= ok
        out[f"range_{rng_ // 1000}s"] = res
    out["parity"] = bool(parity)

    # the new kernels' device time under torch.profiler, in a run of its own (range 300 s, G = 100)
    from torch.profiler import ProfilerActivity, profile
    groups = ((series // nb) % GROUPS[0]).astype(np.uint32)
    n_prof = 5
    eng.scan_histogram_quantile(handle, ins, HG_FN_RATE, series, groups, ubs, QS, [], start, end, STEP_MS, RANGES[0])
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            eng.scan_histogram_quantile(handle, ins, HG_FN_RATE, series, groups, ubs, QS, [], start, end, STEP_MS, RANGES[0])
        torch.cuda.synchronize()
    kus = {}
    for ev in prof.key_averages():
        name = ev.key
        for k in ("histogram_quantile_kernel", "histogram_heads_kernel", "histogram_sort_keys_kernel", "range_function_kernel",
                  "reduce_groups_kernel", "radix"):
            if k in name:
                dev = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                kus[k] = round(kus.get(k, 0.0) + dev / n_prof, 1)
    out["kernels_us_per_call_range_300s_g100"] = kus
    print(json.dumps(out))
    eng.close()
    if not parity:
        sys.exit("the histogram call differs from bucketQuantile over the by-map sums")


if __name__ == "__main__":
    main()
