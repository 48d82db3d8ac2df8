"""Bloom filters on the H100: what writing them costs, and what they save on point lookups.  Prints one JSON line.

(a) Writer cost: tools/bench_compaction.py's default inputs (16 overlapping SSTs, 4000 series x 1000 points, keep 0.5) compacted through
    hg_compact_to_sst with filters on 0, 1 and 2 columns (parquet-rs's default 1 MiB bitset per chunk): wall time, gpu_ms, file size, and
    bloom_build_kernel's own time from a separate torch.profiler run.  `ptxas -v` of the kernel (registers, spills) when nvcc is present.
(b) Lookups: an event table sorted by (host, ts) with a random unique u64 request_id, `events` rows in 16 PK-disjoint SSTs written by the
    GPU writer with a filter on request_id.  `request_id = X` and `request_id IN (8 ids)` through scan (general pipeline), scan_aggregate
    as the engine plans it (`path` bit 0 says whether the fused path ran) and scan_aggregate on the general pipeline, resident and transient, with and without HG_FLAG_NO_BLOOM_FILTER: rows_decoded, gpu_ms, wall; results checked
    against the CPU oracle.  `gpu` names the card and its power limit (nvidia-smi, read only).

Usage: bench_bloom.py [events=32000000]"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

EVENTS = int(sys.argv[1]) if len(sys.argv) > 1 else 32_000_000
NFILES = 16


def median_run(fn, reps=5):
    r = []
    for _ in range(reps):
        t = time.perf_counter()
        st = fn()
        r.append(((time.perf_counter() - t) * 1e3, st["gpu_ms"], st["rows_decoded"], st["path"], st["kernel_launches"]))
    a = np.array(r[1:], dtype=np.float64)
    return {"wall_ms": float(np.median(a[:, 0])), "gpu_ms": float(np.median(a[:, 1])), "rows_decoded": int(r[-1][2]), "path": int(r[-1][3]),
            "kernel_launches": int(r[-1][4])}


def writer_cost(tmp):
    from concurrent.futures import ProcessPoolExecutor
    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import Engine, SchemaHandle, SstInput
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    with ProcessPoolExecutor(max_workers=16) as ex:
        ssts = list(ex.map(_compaction_input, range(16)))
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    names = schema.arrow_schema.names
    eng = Engine(device=0)
    inputs = []
    for data, n, seq in ssts:
        eng.load_sst(handle, SstInput(id=seq, data=data, num_rows=n))
        inputs.append(SstInput(id=seq, num_rows=n, time_start=0, time_end=1, max_sequence=seq))
    path = os.path.join(tmp, "c.sst")
    out = {}
    for label, cols in (("none", ()), ("value", ("value",)), ("series_id+value", ("series_id", "value"))):
        blooms = [n in cols for n in names] if cols else None

        def call():
            meta = eng.compact_to_sst(handle, inputs, path, bloom_filters=blooms)
            st = eng.stats()
            st["file_bytes"] = meta.size
            return st
        r = median_run(call, 4)
        r["file_bytes"] = os.path.getsize(path)
        out[label] = r
    # bloom_build_kernel alone, in a profiled run of its own
    import torch
    from torch.profiler import ProfilerActivity, profile
    blooms = [n in ("series_id", "value") for n in names]
    eng.compact_to_sst(handle, inputs, path, bloom_filters=blooms)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            eng.compact_to_sst(handle, inputs, path, bloom_filters=blooms)
        torch.cuda.synchronize()
    ks = [e for e in prof.key_averages() if "bloom_build_kernel" in e.key]
    out["bloom_build_kernel_ms_per_call"] = (sum(e.device_time_total for e in ks) / 3 / 1e3) if ks else None
    out["rows_out"] = int(eng.compact_to_sst(handle, inputs, path).num_rows)
    eng.close()
    return out


def _compaction_input(f):
    from horaedb_b200 import sstgen
    return sstgen.synth_overlapping_ssts(1, 4000, 1000, 1000, 0.5, compression="snappy", base_seq=1000 + f)[0]


def ptxas_report():
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        return "not measured (no nvcc)"
    csrc = os.path.join(ROOT, "horaedb_b200", "csrc")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "-Xptxas", "-v",
                            "-c", os.path.join(csrc, "sst_writer.cu"), "-o", os.path.join(d, "w.o")], capture_output=True, text=True)
        lines = r.stderr.splitlines()
    out = []
    for i, l in enumerate(lines):
        if "Compiling entry function" in l and "bloom_build" in l:
            out += [x.strip() for x in lines[i + 1:i + 4] if "ptxas info" in x]
    return out or "not measured (no ptxas output for bloom_build_kernel)"


def lookups(tmp):
    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_FLAG_NO_BLOOM_FILTER, HG_FLAG_NO_FUSED, Engine, SchemaHandle, SstInput
    from horaedb_b200.types import StorageSchema
    from oracle import oracle
    import pyarrow as pa
    user = pa.schema([pa.field("host", pa.uint64()), pa.field("ts", pa.int64()), pa.field("request_id", pa.uint64()), pa.field("value", pa.float64())])
    st = StorageSchema.try_new(user, 2)
    handle = SchemaHandle(st.arrow_schema, 2)
    blooms = [n == "request_id" for n in st.arrow_schema.names]
    rng = np.random.default_rng(42)
    per = EVENTS // NFILES
    with np.errstate(over="ignore"):                     # an odd multiplier mod 2^64 keeps the ids unique
        rid_all = rng.permutation(np.arange(1, EVENTS + 1, dtype=np.uint64)) * np.uint64(0x9E3779B97F4A7C15)
    eng = Engine(device=0)
    datas = []
    for f in range(NFILES):
        host = (np.arange(per) // 20_000 + f * 10_000).astype(np.uint64)
        ts = (np.arange(per) % 20_000).astype(np.int64) * 1000
        batch = pa.RecordBatch.from_arrays([pa.array(host), pa.array(ts), pa.array(rid_all[f * per:(f + 1) * per]),
                                            pa.array(rng.standard_normal(per))], schema=user)
        path = os.path.join(tmp, f"e{f}.sst")
        eng.write_batch(handle, batch, 100 + f, path, bloom_filters=blooms)
        with open(path, "rb") as fh:
            datas.append(fh.read())
        os.unlink(path)
    target = int(rid_all[per * 7 + 12_345])
    ids8 = [int(x) for x in rid_all[rng.choice(EVENTS, 8, replace=False)]]
    queries = {"eq": [("request_id", "eq", target)], "in8": [("request_id", "in", ids8)]}
    out = {"rows": EVENTS, "files": NFILES, "file_bytes_total": sum(len(d) for d in datas)}
    rid_keys = [100 + f for f in range(NFILES)]
    for i, d in enumerate(datas):
        eng.load_sst(handle, SstInput(id=rid_keys[i], data=d))
    for residency in ("resident", "transient"):
        seq = iter(range(10_000_000, 20_000_000))
        for qname, preds in queries.items():
            for mode in ("scan_general", "aggregate_auto", "aggregate_general"):
                for bloom in (True, False):
                    flags = (0 if bloom else HG_FLAG_NO_BLOOM_FILTER) | (HG_FLAG_NO_FUSED if mode != "aggregate_auto" else 0)
                    eng.set_flags(flags)

                    def call():
                        ssts = [SstInput(id=rid_keys[i]) for i in range(NFILES)] if residency == "resident" else \
                               [SstInput(id=next(seq), data=d) for d in datas]
                        if mode == "scan_general":
                            res = pa.Table.from_batches(list(eng.scan(handle, ssts, preds, None, False)), schema=user)
                        else:
                            res = eng.scan_aggregate(handle, ssts, preds, group_col=0, ts_col=1, window_ms=60_000, value_col=3)
                        s = eng.stats()
                        s["_rows"] = res.num_rows
                        return s
                    r = median_run(call)
                    out[f"{residency}/{qname}/{mode}/{'bloom' if bloom else 'no_bloom'}"] = r
    eng.set_flags(0)
    # parity with the CPU oracle on the two queries
    for qname, preds in queries.items():
        want = oracle.scan_aggregate(datas, st.arrow_schema, 2, preds, group_col=0, ts_col=1, window_ms=60_000, value_col=3)
        got = eng.scan_aggregate(handle, [SstInput(id=k) for k in rid_keys], preds, group_col=0, ts_col=1, window_ms=60_000, value_col=3)
        ok = got["host"].to_numpy().tolist() == want.gkey.tolist() and got["count"].to_numpy().tolist() == want.count.tolist() and \
            np.array_equal(got["sum"].to_numpy(), want.sum)
        out[f"parity/{qname}"] = bool(ok) and int(want.count.sum()) == (1 if qname == "eq" else 8)
    eng.close()
    return out


if __name__ == "__main__":
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        gpu = "unknown"
    res = {"gpu": gpu}
    with tempfile.TemporaryDirectory() as tmp:
        for name, fn in (("writer", lambda: writer_cost(tmp)), ("ptxas_bloom_build_kernel", ptxas_report), ("lookups", lambda: lookups(tmp))):
            try:
                res[name] = fn()
            except Exception as ex:                     # report what was measured; the failure is part of the result
                res[name] = f"failed: {type(ex).__name__}: {ex}"
    print(json.dumps(res))
