"""Set-membership predicates on the H100: `series_id IN_SET (k series) AND ts in [a, b)`, `sum(value), count` per series, on resident
SSTs of bench.py's config-2 shape (6 250 series x 1 000 points per file, Snappy).  Prints one JSON line.

The k ids are drawn without replacement from [0, max(series in the files, 2 k)), unsorted, so the host sorts every set; one more run
hands the k = 1 000 000 set over already sorted, and one puts a set on the unsorted `tag` column (tag = series_id mod 16).  Per k,
median and [min, max] of `runs` calls after a warm-up:
  * the call's wall time, gpu_ms, rows_decoded / rows_filtered / groups, kernel launches;
  * eval_in_set_kernel's own time from a torch.profiler run of its own, with the bytes it must move at least (8-byte key + 1 alive
    byte written per decoded row, + 1 alive byte read behind the time-range kernel) and their share of 3.35 TB/s;
  * the host's share, from the library's HORAE_TRACE lines of the same calls: conversion + sorted check (+ sort) of the set, and the
    statistics pruning of all files;
  * the same answer by the routes a caller has without the operator: HG_OP_IN at k = 64; beyond, a scan of the enclosing series_id
    range with the time range (projection series_id, value) filtered and grouped on the host with numpy.isin.
Exits non-zero when a count differs between the routes (sums: relative 1e-9, the host adds in another order).  `gpu` names the card
and its power limit (nvidia-smi, read only).

Usage: bench_in_set.py [files=8] [runs=5]"""
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
os.environ["HORAE_TRACE"] = "1"                       # read once by the library: its planning lines go to stderr, redirected below

import bench as shape                                  # noqa: E402  (config-2 generator)

FILES = int(sys.argv[1]) if len(sys.argv) > 1 else 8
RUNS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
KERNEL = "eval_in_set_kernel"
KS = [64, 1_000, 32_000, 1_000_000]


class StderrCapture:
    """the process's fd 2 into a temporary file for the length of a block (the library writes its trace lines with fprintf)"""

    def __enter__(self):
        self.tmp = tempfile.TemporaryFile(mode="w+b")
        sys.stderr.flush()
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


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import Engine, SchemaHandle, SstInput
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    files = shape.gen_ssts(0, "snappy", FILES, min(16, os.cpu_count() or 1))
    if not torch.cuda.is_available():
        sys.exit("bench_in_set.py needs a GPU")
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    ins = []
    for seq, data, n in files:
        eng.load_sst(handle, SstInput(id=seq, data=data))
        ins.append(SstInput(id=seq, num_rows=n))
    n_series = FILES * shape.SERIES_PER_FILE
    span = shape.POINTS * shape.DELTA_MS
    trange = [("ts", "ge", sstgen.T0_MS + span // 4), ("ts", "lt", sstgen.T0_MS + 3 * span // 4)]
    kw = dict(group_col=0, ts_col=-1, window_ms=0, value_col=2)
    rng = np.random.default_rng(42)
    ok = True

    def measure(preds):
        eng.scan_aggregate(handle, ins, preds, **kw)
        wall, gms = [], []
        with StderrCapture() as cap:
            for _ in range(RUNS):
                t = time.perf_counter()
                out = eng.scan_aggregate(handle, ins, preds, **kw)
                wall.append((time.perf_counter() - t) * 1e3)
                gms.append(eng.stats()["gpu_ms"])
        st = eng.stats()
        r = {"wall_ms": _spread(wall), "gpu_ms": _spread(gms), "rows_decoded": st["rows_decoded"], "rows_filtered": st["rows_filtered"],
             "groups": out.num_rows, "kernel_launches": st["kernel_launches"], "path": st["path"]}
        prep = [float(x) for x in re.findall(r"\[in_set\] predicate \d+: .*?, ([0-9.]+) us", cap.text)]
        how = re.findall(r"\[in_set\] predicate \d+: .*?, (already sorted|sorted on the host),", cap.text)
        plan = [float(x) for x in re.findall(r"\[plan\] statistics pruning of \d+ files: ([0-9.]+) us", cap.text)]
        if prep:
            r["host_set_prepare_us"] = _spread(prep)
            r["host_set_order"] = how[0]
        if plan:
            r["host_pruning_us"] = _spread(plan)
        return r, out

    def profiled(preds, rows):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.scan_aggregate(handle, ins, preds, **kw)
            torch.cuda.synchronize()
        kt = sum(getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0)) for ev in prof.key_averages() if KERNEL in ev.key) / 1e3
        moved = rows * (8 + 1 + 1)
        r = {"probe_kernel_ms": round(kt, 4), "probe_kernel_min_bytes": moved}
        if kt > 0:
            r["probe_kernel_GBps"] = round(moved / (kt / 1e3) / 1e9, 1)
            r["probe_kernel_share_of_3.35TBps"] = round(moved / (kt / 1e3) / 3.35e12, 4)
        return r

    def host_route(ids):
        """range scan + numpy.isin + group by on the host"""
        import pyarrow as pa
        preds = [("series_id", "ge", int(ids.min())), ("series_id", "le", int(ids.max())), *trange]
        t = time.perf_counter()
        tbl = pa.Table.from_batches(list(eng.scan(handle, ins, preds, projection=[0, 2])))
        scan_ms = (time.perf_counter() - t) * 1e3
        st = eng.stats()
        sid, val = tbl["series_id"].to_numpy(), tbl["value"].to_numpy()
        m = np.isin(sid, ids)
        keys, start, cnt = np.unique(sid[m], return_index=True, return_counts=True)
        sums = np.add.reduceat(val[m], start) if len(start) else np.zeros(0)
        return {"wall_ms": round((time.perf_counter() - t) * 1e3, 1), "scan_wall_ms": round(scan_ms, 1), "rows_to_host": tbl.num_rows,
                "rows_decoded": st["rows_decoded"]}, keys, cnt, sums

    res = {}
    for k in KS:
        ids = rng.choice(max(n_series, 2 * k), size=k, replace=False).astype(np.uint64)
        preds = [("series_id", "in_set", ids), *trange]
        r, out = measure(preds)
        r.update(profiled(preds, r["rows_decoded"]))
        if k == 64:
            r["HG_OP_IN"], out_in = measure([("series_id", "in", ids.tolist()), *trange])
            same = out.equals(out_in)
            r["HG_OP_IN"]["same_result"] = same
            ok = ok and same
        h, keys, cnt, sums = host_route(ids)
        same = (out["series_id"].to_numpy().tolist() == keys.tolist() and out["count"].to_numpy().tolist() == cnt.tolist()
                and np.allclose(out["sum"].to_numpy(), sums, rtol=1e-9, atol=0))
        h["same_result"] = bool(same)
        ok = ok and same
        r["range_scan_plus_host_isin"] = h
        if k == KS[-1]:
            r["set_already_sorted"], out2 = measure([("series_id", "in_set", np.sort(ids)), *trange])
            ok = ok and out2.equals(out)
        res[f"k={k}"] = r
    tags = np.concatenate([[3, 7], 16 + rng.choice(64_000, size=31_998, replace=False)]).astype(np.uint32)
    rng.shuffle(tags)
    preds = [("tag", "in_set", tags), *trange]
    r, out = measure(preds)
    r.update(profiled(preds, r["rows_decoded"]))
    ref = eng.scan_aggregate(handle, ins, [("tag", "in", [3, 7]), *trange], **kw)
    r["same_result_as_IN"] = out.equals(ref)
    ok = ok and r["same_result_as_IN"]
    res["tag k=32000"] = r
    r, _ = measure(trange)
    res["time range only (fused path)"] = r
    eng.close()
    print(json.dumps({"gpu": gpu, "files": FILES, "rows": sum(n for _, _, n in files), "series": n_series, "runs": RUNS, "all_routes_agree": ok, "results": res}))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
