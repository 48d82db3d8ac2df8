"""`topk(10, rate(x[300s])) by (series % G)` every 60 s on the H100: today's host route against `hg_scan_range_function_topk`.  Prints
one JSON line.

Files and grid: those of tools/bench_range_function.py (16 resident SSTs of 6 250 series x 1 000 points, 10 s apart, uncompressed, 100 M
rows, 100 000 series; every 60 s over the data's whole span), range 300 s, k = 10, label groups series_id % G for G = 1 and 100.  Per
route, the median and [min, max] of `runs` calls after a warm-up, each returning its table:
  (a) host: hg_scan_range_function(HG_FN_RATE), one value per series and step, then top-k per (group, t) in numpy (a stable lexsort by
            (group, t, NaN, -value) and the first k of each segment);
  (b) topk: hg_scan_range_function_topk(HG_FN_RATE, k = 10), at most k rows per (group, t).
gpu_ms is the call's device time (the engine's events, the result's copy to the host included); wall_ms the host's time for the whole
route (for (a) with its numpy part).  `parity`: (b)'s rows equal (a)'s, values bit for bit.  `profile`: a separate torch.profiler run of
(b) at G = 100: the device time of its top-k kernels and the share of the call's kernel time taken by the radix sort's histogram and
scatter kernels (the value pass and the (group, t) pass).  `gpu` names the card and its power limit (nvidia-smi, read only).

Usage: bench_range_topk.py [files=16] [runs=5] [out_dir]"""
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
OUT_DIR = sys.argv[3] if len(sys.argv) > 3 else None
STEP_MS, RANGE_MS, K = 60_000, 300_000, 10
GROUPS = (1, 100)


def _spread(xs):
    return {"median": round(float(np.median(xs)), 3), "min": round(float(min(xs)), 3), "max": round(float(max(xs)), 3)}


def host_topk(per, G, k):
    """top-k per (series % G, t) of the per-series table: value descending, NaN last, ties in series order (the input's order)"""
    sid = per["series_id"].to_numpy()
    t = per["t"].to_numpy()
    v = per["value"].to_numpy()
    g = (sid % G).astype(np.uint32)
    nan = np.isnan(v)
    neg = np.where(nan, 0.0, -(v + 0.0))
    order = np.lexsort((neg, nan, t, g))               # stable: equal keys keep (series, t) order
    gs, ts = g[order], t[order]
    head = np.ones(len(order), bool)
    head[1:] = (gs[1:] != gs[:-1]) | (ts[1:] != ts[:-1])
    starts = np.flatnonzero(head)
    rank = np.arange(len(order)) - np.repeat(starts, np.diff(np.append(starts, len(order))))
    keep = order[rank < k]
    return g[keep], t[keep], sid[keep], v[keep]


def main():
    import torch

    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_FN_RATE, HG_TOPK, Engine, SchemaHandle, SstInput
    shape.SERIES_PER_FILE, shape.POINTS, shape.DELTA_MS = 6250, 1000, 10_000
    files = shape.gen_ssts(0, "none", FILES, min(16, os.cpu_count() or 1))
    if not torch.cuda.is_available():
        sys.exit("bench_range_topk.py needs a GPU")
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

    out = {"workload": f"topk({K}, rate(x[{RANGE_MS // 1000}s])) by (series % G) every {STEP_MS // 1000} s: {FILES} resident SSTs, {rows} rows, "
                       "uncompressed", "gpu": gpu, "rows": rows, "runs": RUNS, "grid": {"start_ms": start, "end_ms": end, "step_ms": STEP_MS}}
    series = None
    parity = True
    for G in GROUPS:
        res = {}

        def host_route():
            per = eng.scan_range_function(handle, ins, HG_FN_RATE, [], start, end, STEP_MS, RANGE_MS)
            host_route.d2h = eng.stats()["bytes_d2h"]
            host_route.gpu_ms = eng.stats()["gpu_ms"]
            return per, host_topk(per, G, K)
        (per, exp), res["a_host"] = timed(host_route)
        res["a_host"]["bytes_d2h"] = host_route.d2h
        res["a_host"]["rows_out"] = int(len(exp[0]))
        series = np.unique(per["series_id"].to_numpy())
        groups = (series % G).astype(np.uint32)
        got, res["b_topk"] = timed(lambda: eng.scan_range_function_topk(handle, ins, HG_FN_RATE, K, series, groups, [], start, end, STEP_MS,
                                                                         RANGE_MS, order=HG_TOPK))
        ok = got.num_rows == len(exp[0])
        ok = ok and bool(np.array_equal(got["group"].to_numpy(), exp[0])) and bool(np.array_equal(got["t"].to_numpy(), exp[1]))
        ok = ok and bool(np.array_equal(got["series_id"].to_numpy(), exp[2]))
        ok = ok and bool(np.array_equal(got["value"].to_numpy().view(np.uint64), exp[3].view(np.uint64)))
        res["b_topk"]["parity"] = ok
        parity &= ok
        out[f"g{G}"] = res
    out["parity"] = bool(parity)

    # a separate profiled run: the top-k kernels and the two radix sorts' share of the call's kernel time
    from torch.profiler import ProfilerActivity, profile
    groups = (series % GROUPS[-1]).astype(np.uint32)
    call = lambda: eng.scan_range_function_topk(handle, ins, HG_FN_RATE, K, series, groups, [], start, end, STEP_MS, RANGE_MS)  # noqa: E731
    call()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(RUNS):
            call()
        torch.cuda.synchronize()
    per_kernel = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and "CUDA" in str(ev.device_type) and ev.count:
            per_kernel[ev.key] = per_kernel.get(ev.key, 0.0) + ev.self_device_time_total / RUNS / 1e3
    kernels = {k: v for k, v in per_kernel.items() if "memcpy" not in k.lower() and "memset" not in k.lower()}
    total = sum(kernels.values())
    radix = sum(v for k, v in kernels.items() if "radix_" in k)
    topk = {k.split("(")[0].split("::")[-1]: round(v, 4) for k, v in kernels.items() if "topk_" in k}
    out["profile"] = {"g": GROUPS[-1], "kernel_ms_per_call": round(total, 3), "radix_sort_ms_per_call": round(radix, 3),
                      "radix_sort_share": round(radix / total, 3) if total else None, "topk_kernels_ms_per_call": topk}
    if OUT_DIR:
        os.makedirs(OUT_DIR, exist_ok=True)
        with open(os.path.join(OUT_DIR, "bench_range_topk_kernels.json"), "w") as f:
            json.dump({k: round(v, 4) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])}, f, indent=1)
    print(json.dumps(out))
    eng.close()
    if not parity:
        sys.exit("the top-k call differs from the host's top-k of the per-series values")


if __name__ == "__main__":
    main()
