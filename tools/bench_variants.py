"""Developer tool: time the fused scan kernel with (0) and without (1) the late-materialisation gate
(HG_FLAG_NO_LATE_MATERIALIZATION) on the config-2 workload, one process each."""
import multiprocessing as mp
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def run(variant, ssts, steps):
    import numpy as np
    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import HG_FLAG_NO_LATE_MATERIALIZATION, Engine, SchemaHandle, SstInput
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    if variant:
        eng.set_flags(HG_FLAG_NO_LATE_MATERIALIZATION)
    for sid, data, n in ssts:
        eng.load_sst(handle, SstInput(id=sid, data=data, num_rows=n))
    res = [SstInput(id=sid, num_rows=n) for sid, _, n in ssts]
    P = bench.preds()
    km, gm, wall = [], [], []
    for it in range(steps + 3):
        t = time.perf_counter()
        eng.scan_aggregate_device(handle, res, P, group_col=0, ts_col=-1, window_ms=0, value_col=2)
        w = time.perf_counter() - t
        st = eng.stats()
        if it >= 3:
            km.append(st["kernel_ms"]); gm.append(st["gpu_ms"]); wall.append(w * 1e3)
    rows = st["rows_decoded"]
    print(f"{'ungated' if variant else 'gated'}: kernel {np.median(km):.3f} ms  call(gpu) {np.median(gm):.3f} ms  wall {np.median(wall):.3f} ms  "
          f"-> {rows * 28 / np.median(km) / 1e6:.0f} GB/s (28 B/row) on {rows} decoded rows, {st['rows_materialized']} materialised, "
          f"groups {st['groups_out']}", flush=True)
    # other query shapes on the same data (kernel_ms only)
    for name, kw, pr in (("count(*)", dict(group_col=-1, ts_col=-1, window_ms=0, value_col=-1), []),
                         ("sum per series, no filter", dict(group_col=0, ts_col=-1, window_ms=0, value_col=2), []),
                         ("1-min buckets, filter", dict(group_col=0, ts_col=1, window_ms=60000, value_col=2), P)):
        ks = []
        for it in range(4):
            eng.scan_aggregate_device(handle, res, pr, **kw)
            ks.append(eng.stats()["kernel_ms"])
        st = eng.stats()
        print(f"    {name}: kernel {min(ks):.3f} ms path={st['path']} rows_decoded={st['rows_decoded']} materialised={st['rows_materialized']} groups={st['groups_out']}", flush=True)
    eng.close()


if __name__ == "__main__":
    variants = [int(x) for x in sys.argv[1].split(",")] if len(sys.argv) > 1 else [0, 1]
    nfiles = int(sys.argv[2]) if len(sys.argv) > 2 else 16
    ssts = bench.gen_ssts(0, "none", nfiles, min(os.cpu_count(), 16))
    for v in variants:
        p = mp.get_context("fork").Process(target=run, args=(v, ssts, 10))
        p.start()
        p.join()
