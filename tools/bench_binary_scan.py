"""Binary columns on the H100 by encoding: the same Append-mode table written PLAIN, DELTA_LENGTH_BYTE_ARRAY, dictionary and DELTA_BYTE_ARRAY,
scanned resident (hg_scan_open) and merged through hg_compact_open.  Prints one JSON line.

Table: (host u64, ts i64) primary key, a log-like `payload` Binary column (a shared "host-NNNNN/cpu/N/" prefix + random bytes, 40 B) and a
low-cardinality `labels` column; `nfiles` PK-disjoint SSTs plus `nfiles` SSTs that overlap them, `rows` rows each, Snappy pages.  Per
encoding: wall time, gpu_ms, kernel_ms and rows/s (median of 3 after one warm-up), and the kernels' own times from a separate
torch.profiler run (decode_chunks_kernel, dba_materialise_kernel) with the DELTA_BYTE_ARRAY kernel's materialised bytes per second.  The
four outputs must be identical (SHA-256 of the Arrow buffers); the tool exits non-zero otherwise.  `gpu` names the card and its power
limit (nvidia-smi, read only).

Usage: bench_binary_scan.py [rows=1000000] [nfiles=16]"""
import hashlib
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

ROWS = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
NFILES = int(sys.argv[2]) if len(sys.argv) > 2 else 16
ENCODINGS = ["PLAIN", "DELTA_LENGTH_BYTE_ARRAY", "DICTIONARY", "DELTA_BYTE_ARRAY"]


def _schema():
    import pyarrow as pa
    from horaedb_b200.types import StorageSchema, UpdateMode
    user = pa.schema([pa.field("host", pa.uint64()), pa.field("ts", pa.int64()), pa.field("payload", pa.binary()), pa.field("labels", pa.binary())])
    return StorageSchema.try_new(user, 2, UpdateMode.Append), user


def _make(f):
    """-> {encoding: SST bytes} of file f: f < NFILES covers its own host range; f >= NFILES overlaps file f - NFILES."""
    import pyarrow as pa
    from horaedb_b200 import sstgen
    from horaedb_b200.config import ColumnOptions, WriteConfig
    schema, user = _schema()
    rng = np.random.default_rng(1000 + f)
    base = f % NFILES
    host = np.sort(rng.integers(0, 10_000, ROWS)).astype(np.uint64) + np.uint64(base * 10_000)
    ts = np.arange(ROWS, dtype=np.int64) * 10 + (f // NFILES) * 5           # overlapping files interleave with their partner's rows
    order = np.lexsort((ts, host))
    host, ts = host[order], ts[order]
    hm = (host % 100_000).astype(np.int64)
    col = lambda b: np.tile(np.frombuffer(b, np.uint8), (ROWS, 1))
    digits = np.stack([(hm // 10 ** k) % 10 + 48 for k in (4, 3, 2, 1, 0)], axis=1).astype(np.uint8)
    pre = np.concatenate([col(b"host-"), digits, col(b"/cpu/"), (host % 4 + 48).astype(np.uint8)[:, None], col(b"/")], axis=1)   # 17 B
    tail = rng.integers(48, 123, (ROWS, 23), dtype=np.uint8)
    vals = np.concatenate([pre, tail], axis=1)                               # 40 B per value
    payload = pa.Array.from_buffers(pa.binary(), ROWS, [None, pa.py_buffer((np.arange(ROWS + 1, dtype=np.int32) * 40).tobytes()), pa.py_buffer(vals.tobytes())])
    lab = [b"env=prod,dc=%d" % i for i in range(8)]
    li = rng.integers(0, 8, ROWS)
    labels = pa.array([lab[i] for i in li], pa.binary())
    batch = pa.RecordBatch.from_arrays([pa.array(host), pa.array(ts), payload, labels], schema=user)
    out = {}
    for enc in ENCODINGS:
        if enc == "DICTIONARY":
            cfg = WriteConfig(enable_dict=True)
        elif enc == "PLAIN":
            cfg = WriteConfig()
        else:
            cfg = WriteConfig(column_options={c: ColumnOptions(encoding=enc) for c in ("payload", "labels")})
        out[enc] = sstgen.write_sst(schema, batch, seq=10 + f, cfg=cfg, presorted=True)
    return out, int(vals.size + sum(len(lab[i]) for i in li))


def _digest(batches):
    import pyarrow as pa
    t = pa.Table.from_batches(batches).combine_chunks()
    h = hashlib.sha256()
    for c in t.columns:
        for b in c.chunks[0].buffers():
            if b is not None:
                h.update(b.to_pybytes())
    return h.hexdigest()


def main():
    import torch
    from horaedb_b200._ffi import Engine, SchemaHandle, SstInput
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    with ProcessPoolExecutor(max_workers=16) as ex:
        made = list(ex.map(_make, range(2 * NFILES)))
    value_bytes = sum(b for _, b in made)
    schema, _ = _schema()
    from horaedb_b200.types import UpdateMode
    handle = SchemaHandle(schema.arrow_schema, 2, UpdateMode.Append)
    eng = Engine(device=0)
    res, digests = {}, {}
    for e_i, enc in enumerate(ENCODINGS):
        ids = []
        for f, (files, _) in enumerate(made):
            ids.append(1_000 * (e_i + 1) + f)
            eng.load_sst(handle, SstInput(id=ids[-1], data=files[enc]))
        ins = [SstInput(id=i) for i in ids]
        r = {"file_mb": round(sum(len(files[enc]) for files, _ in made) / 1e6, 1)}
        for label, fn in (("scan", lambda: list(eng.scan(handle, ins))), ("compact", lambda: list(eng.compact(handle, ins)))):
            out = fn()                                                       # warm-up
            digests.setdefault(label, {})[enc] = _digest(out)
            del out
            runs = []
            for _ in range(3):
                t = time.perf_counter()
                out = fn()
                wall = (time.perf_counter() - t) * 1e3
                st = eng.stats()
                runs.append((wall, st["gpu_ms"], st["kernel_ms"], st["rows_in_files"]))
                del out
            a = np.median(np.array(runs, dtype=np.float64), axis=0)
            r[label] = {"wall_ms": round(float(a[0]), 2), "gpu_ms": round(float(a[1]), 2), "kernel_ms": round(float(a[2]), 2),
                        "rows_per_s": round(float(a[3]) / (float(a[0]) / 1e3), 0)}
        # kernels' own times, in a run of their own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            list(eng.scan(handle, ins))
            torch.cuda.synchronize()
        ks = {}
        for ev in prof.key_averages():
            for k in ("decode_chunks_kernel", "dba_materialise_kernel"):
                if k in ev.key:
                    ks[k] = round(getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0)) / 1e3, 3)
        r["kernel_time_ms"] = ks
        if "dba_materialise_kernel" in ks and ks["dba_materialise_kernel"] > 0:
            bps = value_bytes / (ks["dba_materialise_kernel"] / 1e3)
            r["dba_materialised_GBps"] = round(bps / 1e9, 1)
            r["dba_share_of_3.35TBps"] = round(bps / 3.35e12, 4)
        res[enc] = r
        for i in ids:
            eng.unload_sst(i)
    eng.close()
    same = all(len(set(d.values())) == 1 for d in digests.values())
    print(json.dumps({"gpu": gpu, "rows_per_file": ROWS, "files": 2 * NFILES, "value_bytes": value_bytes, "outputs_identical": same, "results": res}))
    if not same:
        print(json.dumps(digests), file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
