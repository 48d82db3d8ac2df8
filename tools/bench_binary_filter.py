"""Predicates on Binary columns on the H100: eval_binary_predicates_kernel and the calls around it, per Binary encoding.  Prints one JSON
line.

Table: the shape of tools/bench_binary_scan.py — (host u64, ts i64) primary key, a 40-byte `payload` ("host-NNNNN/cpu/N/" shared 17-byte
prefix + random bytes) and a dictionary-friendly `labels` column (8 values) — `nfiles` PK-disjoint Append-mode SSTs of `rows` rows each,
resident, written PLAIN, DELTA_LENGTH_BYTE_ARRAY, dictionary and DELTA_BYTE_ARRAY.  The files are disjoint and their keys unique, so the
merge keeps every row and the filtered scan equals an unfiltered scan filtered afterwards: today's only way to the answer, a full scan
plus a `pyarrow.compute` filter on the host.

Queries: `labels = x`; `payload >= a AND payload < b` (bounds sharing the first 8 bytes with the rows of 1 % of the hosts, which need the
compare past the key); `payload IN (8 values)`.  Per query and encoding (median of 3 after a warm-up):
  * the call's wall time and gpu_ms, against the same scan without the predicate, and against the unfiltered scan + host filter;
  * rows_decoded with pruning on and off;
  * the predicate kernel's own time from a torch.profiler run of its own, with pruning on and off (off: every row reaches the kernel),
    with the bytes it must move at least (per row: the value pointer 8 B, length 4 B, validity 1 B, alive byte 1 B, the value's first
    8 bytes) and their share of 3.35 TB/s.
Exits non-zero if a filtered result differs from the host-filtered one (Table.equals: values, validity, order).  `gpu` names the card and its
power limit (nvidia-smi, read only).

Usage: bench_binary_filter.py [rows=1000000] [nfiles=8]"""
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_binary_scan as shape                      # noqa: E402  (table generator: reads ROWS / NFILES from its module globals)

ROWS = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
NFILES = int(sys.argv[2]) if len(sys.argv) > 2 else 8
shape.ROWS, shape.NFILES = ROWS, NFILES
KERNEL = "eval_binary_predicates_kernel"


def _make(f):
    shape.ROWS, shape.NFILES = ROWS, NFILES          # worker processes
    return shape._make(f)


def _host_filter(table, preds):
    import pyarrow as pa
    import pyarrow.compute as pc
    ops = {"eq": pc.equal, "lt": pc.less, "ge": pc.greater_equal}
    m = None
    for col, op, lit in preds:
        x = pc.is_in(table[col], value_set=pa.array(lit, pa.binary())) if op == "in" else ops[op](table[col], pa.scalar(lit, pa.binary()))
        m = x if m is None else pc.and_(m, x)
    return table.filter(pc.fill_null(m, False))


def main():
    import pyarrow as pa
    import pyarrow.parquet as pq
    import torch
    from torch.profiler import ProfilerActivity, profile

    from horaedb_b200._ffi import HG_FLAG_NO_PRUNING, Engine, SchemaHandle, SstInput
    from horaedb_b200.types import UpdateMode
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    with ProcessPoolExecutor(max_workers=16) as ex:
        made = list(ex.map(_make, range(NFILES)))              # f < NFILES: disjoint host ranges
    schema, _ = shape._schema()
    handle = SchemaHandle(schema.arrow_schema, 2, UpdateMode.Append)
    t0 = pq.read_table(io.BytesIO(made[0][0]["PLAIN"]), columns=["payload"])["payload"].to_pylist()
    sample = [t0[i] for i in np.random.default_rng(5).integers(0, len(t0), 7)] + [b"host-99999/cpu/9/not-there"]
    queries = {"labels_eq": [("labels", "eq", b"env=prod,dc=3")],
               "payload_range": [("payload", "ge", b"host-00050/cpu/1/"), ("payload", "lt", b"host-00050/cpu/3/")],
               "payload_in8": [("payload", "in", sample)]}
    eng = Engine(device=0)
    res, ok = {}, True

    def timed(fn, n=3):
        fn()
        runs = []
        for _ in range(n):
            t = time.perf_counter()
            out = fn()
            wall = (time.perf_counter() - t) * 1e3
            st = eng.stats()
            runs.append((wall, st["gpu_ms"]))
            del out
        a = np.median(np.array(runs), axis=0)
        return round(float(a[0]), 2), round(float(a[1]), 2)

    for e_i, enc in enumerate(shape.ENCODINGS):
        ids = []
        for f, (files, _) in enumerate(made):
            ids.append(1_000 * (e_i + 1) + f)
            eng.load_sst(handle, SstInput(id=ids[-1], data=files[enc]))
        ins = [SstInput(id=i) for i in ids]
        scan = lambda preds: pa.Table.from_batches(list(eng.scan(handle, ins, preds)), schema=schema.user_schema())
        full_wall, full_gpu = timed(lambda: scan([]))
        r = {"unfiltered_scan": {"wall_ms": full_wall, "gpu_ms": full_gpu}}
        for qn, preds in queries.items():
            q = {}
            q["wall_ms"], q["gpu_ms"] = timed(lambda: scan(preds))
            st = eng.stats()
            q["rows_decoded"], q["rows_filtered"] = st["rows_decoded"], st["rows_filtered"]
            got = scan(preds)
            host_wall, _ = timed(lambda: _host_filter(scan([]), preds))
            want = _host_filter(scan([]), preds)
            same = got.num_rows == want.num_rows and got.equals(want)
            ok = ok and same
            q["rows_out"], q["matches_host_filter"] = got.num_rows, same
            q["unfiltered_scan_plus_host_filter_wall_ms"] = host_wall
            eng.set_flags(HG_FLAG_NO_PRUNING)
            scan(preds)
            q["rows_decoded_no_pruning"] = eng.stats()["rows_decoded"]
            eng.set_flags(0)
            for suffix, flags, rows in (("", 0, q["rows_decoded"]), ("_no_pruning", HG_FLAG_NO_PRUNING, q["rows_decoded_no_pruning"])):
                eng.set_flags(flags)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    scan(preds)
                    torch.cuda.synchronize()
                eng.set_flags(0)
                kt = sum(getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0)) for ev in prof.key_averages() if KERNEL in ev.key) / 1e3
                moved = rows * (8 + 4 + 1 + 1 + 8)                  # payload 40 B, labels 14 B: both read their whole 8-byte key
                q["kernel_ms" + suffix] = round(kt, 3)
                q["kernel_min_bytes" + suffix] = moved
                if kt > 0:
                    q["kernel_GBps" + suffix] = round(moved / (kt / 1e3) / 1e9, 1)
                    q["kernel_share_of_3.35TBps" + suffix] = round(moved / (kt / 1e3) / 3.35e12, 4)
            r[qn] = q
        res[enc] = r
        for i in ids:
            eng.unload_sst(i)
    eng.close()
    print(json.dumps({"gpu": gpu, "rows_per_file": ROWS, "files": NFILES, "all_match_host_filter": ok, "results": res}))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
