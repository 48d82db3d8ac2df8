"""Config-5 measurement (SURVEY 8d): k overlapping SSTs of one segment -> one sorted, deduplicated run
(hg_compact_open = Executor::do_compaction's plan, keep_builtin), and the same through the GPU SST writer (hg_compact_to_sst).
Prints one JSON line.  `compact_to_sst_by_codec` times the GPU writer with each page codec on the same inputs, `host_zstd_path` the path a
Zstd table took before the GPU writer had Zstandard pages (merged result exported to the host, pyarrow writes the file),
`compact_to_sst_by_encoding` the GPU writer with DELTA_BINARY_PACKED / dictionary pages (Snappy) next to the host path those tables took
before (hg_compact_open + pyarrow with the same options), and `gpu` names the card and its power limit (nvidia-smi, read only).

Usage: bench_compaction.py [k=16] [series=4000] [points=1000] [keep=0.5] [codec=snappy] [procs=16]
BASELINE config 5 at size: bench_compaction.py 64 15625 1000 0.25 snappy 32   (64 SSTs x 3.9 M rows = 250 M rows in)"""
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

k = int(sys.argv[1]) if len(sys.argv) > 1 else 16
series = int(sys.argv[2]) if len(sys.argv) > 2 else 4000
points = int(sys.argv[3]) if len(sys.argv) > 3 else 1000
keep = float(sys.argv[4]) if len(sys.argv) > 4 else 0.5
codec = sys.argv[5] if len(sys.argv) > 5 else "snappy"
procs = int(sys.argv[6]) if len(sys.argv) > 6 else 16


def _one(f):
    from horaedb_b200 import sstgen
    return sstgen.synth_overlapping_ssts(1, series, points, 1000, keep, compression=codec, base_seq=1000 + f)[0]


if __name__ == "__main__":
    t0 = time.perf_counter()
    with ProcessPoolExecutor(max_workers=procs) as ex:
        ssts = list(ex.map(_one, range(k)))
    gen_s = time.perf_counter() - t0

    import numpy as np
    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_FLAG_PAIRWISE_MERGE, Engine, SchemaHandle, SstInput

    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    inputs = []
    for i, (data, n, seq) in enumerate(ssts):
        eng.load_sst(handle, SstInput(id=seq, data=data, num_rows=n))
        inputs.append(SstInput(id=seq, num_rows=n, time_start=0, time_end=1, max_sequence=seq))
    rows_in = sum(n for _, n, _ in ssts)
    peak = 3350.0   # H100 SXM HBM3 GB/s, NVIDIA data sheet

    def run(reps=4):
        res = []
        out = None
        for it in range(reps):
            t = time.perf_counter()
            out = eng.compact(handle, inputs).read_all()
            wall = time.perf_counter() - t
            st = eng.stats()
            res.append((st["merge_ms"], st["kernel_ms"], st["gpu_ms"], wall * 1e3))
        return np.median(np.array(res[1:]), axis=0), out, eng.stats()

    m, out, st = run()
    sid, ts = out["series_id"].to_numpy(), out["ts"].to_numpy()
    key = sid.astype(np.uint64) * np.uint64(1 << 32) + (ts - sstgen.T0_MS).astype(np.uint64)
    assert np.all(key[1:] > key[:-1]), "output must be sorted and duplicate-free"
    eng.set_flags(HG_FLAG_PAIRWISE_MERGE)
    mp, outp, _ = run(3)
    assert outp.num_rows == out.num_rows
    eng.set_flags(0)
    # end to end on the GPU: merge + dedup + Parquet encode (Snappy) + file written
    path = os.path.join(tempfile.mkdtemp(), "out.sst")
    wt = []
    for it in range(3):
        t = time.perf_counter()
        meta = eng.compact_to_sst(handle, inputs, path)
        wt.append(((time.perf_counter() - t) * 1e3, eng.stats()["gpu_ms"]))
    wt = np.median(np.array(wt[1:]), axis=0)
    # the GPU writer per page codec, then the host path it replaces for Zstd tables (hg_compact_open + pyarrow/libzstd writer)
    by_codec = {}
    for wc in ("none", "snappy", "zstd"):
        r = []
        for it in range(4):
            t = time.perf_counter()
            wmeta = eng.compact_to_sst(handle, inputs, path, compression=wc)
            r.append(((time.perf_counter() - t) * 1e3, eng.stats()["gpu_ms"]))
        r = np.median(np.array(r[1:]), axis=0)
        by_codec[wc] = {"wall_ms": float(r[0]), "gpu_ms": float(r[1]), "file_bytes": int(wmeta.size)}
    from horaedb_b200.config import WriteConfig
    hp, host_bytes = [], 0
    for it in range(3):
        t = time.perf_counter()
        tbl = eng.compact(handle, inputs).read_all().combine_chunks()
        data = sstgen.write_sst_with_seq(schema, tbl.to_batches()[0], WriteConfig(compression="zstd"))
        with open(path, "wb") as fh:
            fh.write(data)
        hp.append((time.perf_counter() - t) * 1e3)
        host_bytes = len(data)
    host = {"wall_ms": float(np.median(hp[1:])), "file_bytes": host_bytes,
            "path": "eng.compact (merged result to pinned host memory) + sstgen.write_sst_with_seq(compression=zstd, pyarrow default level)"}
    # the GPU writer per encoding configuration (Snappy pages), and the host path those tables took before (hg_compact_open + pyarrow
    # writing the same options)
    import io
    import pyarrow.parquet as pq
    from horaedb_b200.config import ColumnOptions, resolve_column_options
    D = "DELTA_BINARY_PACKED"
    enc_cfgs = {"plain": WriteConfig(),
                "delta_ints": WriteConfig(encoding=D, column_options={"value": ColumnOptions(encoding="PLAIN")}),
                "dict_keys": WriteConfig(column_options={n: ColumnOptions(enable_dict=True) for n in ("series_id", "tag", "__seq__")}),
                "mixed": WriteConfig(column_options={"series_id": ColumnOptions(enable_dict=True), "tag": ColumnOptions(enable_dict=True),
                                                     "ts": ColumnOptions(encoding=D), "__seq__": ColumnOptions(encoding=D)})}

    def column_bytes(data):
        md = pq.ParquetFile(io.BytesIO(data)).metadata
        return {md.schema.column(c).name: sum(md.row_group(g).column(c).total_compressed_size for g in range(md.num_row_groups))
                for c in range(md.num_columns)}
    by_enc = {}
    for name, wcfg in enc_cfgs.items():
        cols = resolve_column_options(wcfg, schema.arrow_schema)
        r = []
        for it in range(4):
            t = time.perf_counter()
            emeta = eng.compact_to_sst(handle, inputs, path, columns=cols)
            r.append(((time.perf_counter() - t) * 1e3, eng.stats()["gpu_ms"]))
        r = np.median(np.array(r[1:]), axis=0)
        with open(path, "rb") as fh:
            gdata = fh.read()
        hp = []
        for it in range(3):
            t = time.perf_counter()
            tbl = eng.compact(handle, inputs).read_all().combine_chunks()
            hdata = sstgen.write_sst_with_seq(schema, tbl.to_batches()[0], wcfg)
            with open(path, "wb") as fh:
                fh.write(hdata)
            hp.append((time.perf_counter() - t) * 1e3)
        by_enc[name] = {"columns": [list(c) for c in cols], "wall_ms": float(r[0]), "gpu_ms": float(r[1]), "file_bytes": int(emeta.size),
                        "column_bytes": column_bytes(gdata),
                        "host_path": {"wall_ms": float(np.median(hp[1:])), "file_bytes": len(hdata), "column_bytes": column_bytes(hdata)}}
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        gpu = "unknown"
    alg = rows_in * 64
    print(json.dumps({"workload": f"merge-compaction: {k} overlapping SSTs, {rows_in} rows in, {out.num_rows} rows out, codec {codec}",
                      "rows_in": rows_in, "rows_out": out.num_rows, "merge_ms": float(m[0]), "decode_ms": float(m[1]), "call_gpu_ms": float(m[2]),
                      "wall_ms": float(m[3]), "merge_rows_per_s": rows_in / (m[0] / 1e3), "call_rows_per_s": rows_in / (m[3] / 1e3),
                      "roofline_merge": {"alg_bytes": alg, "bytes_model": "64 B per input row (SURVEY 8d: read 4 columns incl. __seq__ + write them once)",
                                         "achieved_GBps": alg / (m[0] / 1e3) / 1e9, "peak_GBps": peak, "frac": alg / (m[0] / 1e3) / 1e9 / peak},
                      "pairwise_passes": {"merge_ms": float(mp[0]), "frac": alg / (mp[0] / 1e3) / 1e9 / peak,
                                          "note": "HG_FLAG_PAIRWISE_MERGE: log2(k) merge-path passes over 32-byte records (round 1)"},
                      "compact_to_sst": {"wall_ms": float(wt[0]), "gpu_ms": float(wt[1]), "file_bytes": int(meta.size), "rows": int(meta.num_rows),
                                         "rows_in_per_s": rows_in / (wt[0] / 1e3)},
                      "compact_to_sst_by_codec": by_codec, "host_zstd_path": host, "compact_to_sst_by_encoding": by_enc, "gpu": gpu,
                      "kernel_launches": st["kernel_launches"], "generate_s": gen_s}))
    eng.close()
