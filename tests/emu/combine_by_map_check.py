"""TEST INFRASTRUCTURE: the REDUCE combine (hg_agg_combine, csrc/comm.cu) of by-map partials (hg_scan_aggregate_by_map_device) with WORLD
ranks as threads of this process, each with its own engine of the emulated build (cuda_emu.h) and tests/emu/nccl_emu.cpp standing in for
NCCL, as tests/emu/combine_check.py does for column keys.  Every rank holds its own series; the map sends series of every rank into the
same label groups, so every group crosses ranks.  The combined table must equal the model's multi-shard definition on every rank: per
shard, the group's sequential f64 sum (tests/group_map_model.py); shards added in rank order; counts summed, min / max taken.

    python tests/emu/combine_by_map_check.py WORLD"""
import ctypes as C
import os
import sys
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ.setdefault("HORAE_EMU_CRASH_REPORT", "1")

import numpy as np  # noqa: E402

import build_engine_emu  # noqa: E402
from horaedb_b200 import _ffi  # noqa: E402

_ffi.LIB_PATH = build_engine_emu.build()
_ffi._lib = None

from horaedb_b200 import sstgen  # noqa: E402
from horaedb_b200._ffi import HG_AGG_HASH, HG_AGG_RUNS, HG_COMBINE_REDUCE, Engine, SchemaHandle, SstInput  # noqa: E402
from group_map_model import aggregate_by_map, reduce_shards  # noqa: E402

SERIES_PER_FILE, FILES_PER_RANK = 40, 2
N_GROUPS = 5


def f64bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def to_host(ptr, n):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int64)), shape=(n,)).copy()      # "device" memory of the emulated build


def the_map(world):
    """every other series of every rank, series s into group (s * 7) % N_GROUPS, with 0xFFFFFFFF for every 11th: unsorted"""
    keys = np.arange(0, world * FILES_PER_RANK * SERIES_PER_FILE, 2, dtype=np.uint64)[::-1].copy()
    groups = ((keys * 7) % N_GROUPS).astype(np.uint32)
    groups[keys % 11 == 0] = 0xFFFFFFFF
    return keys, groups


def rank_main(rank, world, uid, all_datas, schema, errors):
    try:
        eng = Engine(device=0)
        eng.comm_init(uid, rank, world)
        handle = SchemaHandle(schema.arrow_schema, 2)
        mine = [SstInput(id=1000 * rank + i, data=d) for i, d in enumerate(all_datas[rank])]
        t0 = sstgen.T0_MS
        preds = [("ts", "ge", t0 + 20_000), ("ts", "lt", t0 + 250_000)]
        keys, groups = the_map(world)
        for window, mode in ((60_000, HG_AGG_HASH), (0, HG_AGG_RUNS)):
            kw = dict(group_col=0, ts_col=1, window_ms=window, value_col=2)
            eng.scan_aggregate_by_map_device(handle, mine, keys, groups, preds, mode=mode, **kw)
            cmb = eng.combine(HG_COMBINE_REDUCE, 0)
            eng.comm_sync()
            G, rc = cmb.num_groups, cmb.reduced_capacity
            tbl = to_host(cmb.d_reduced, 6 * rc).reshape(6, rc)[:, :G]
            shards = [aggregate_by_map(all_datas[r], schema.arrow_schema, 2, preds, 0, keys, groups, 1, window, 2) for r in range(world)]
            acc = reduce_shards(shards)
            ks = sorted(acc)
            assert G == len(ks), (G, len(ks))
            assert all(len({int(g) for g in s["group"].to_pylist()}) == len(set(k[0] for k in ks)) for s in shards), "a group that is not on every rank"
            assert tbl[0].tolist() == [k[0] for k in ks] and tbl[1].tolist() == [k[1] for k in ks]
            assert tbl[2].tolist() == [acc[k][0] for k in ks]
            for j in range(1, 4):
                assert np.array_equal(tbl[2 + j], f64bits(np.array([acc[k][j] for k in ks]))), j
        eng.comm_destroy()
        eng.close()
        print(f"rank {rank}/{world}: combine by map ok", flush=True)
    except BaseException as e:                                   # a failed rank must not leave the others waiting in an all-gather
        errors.append((rank, repr(e)))
        import traceback
        traceback.print_exc()
        os._exit(1)


def main():
    world = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    schema = sstgen.metric_storage_schema()
    per = SERIES_PER_FILE
    all_datas = [[sstgen.synth_sst((r * FILES_PER_RANK + f) * per, (r * FILES_PER_RANK + f + 1) * per, 300, 1000, seq=100 + r * 10 + f,
                                   compression="snappy" if f % 2 == 0 else "none")[0] for f in range(FILES_PER_RANK)] for r in range(world)]
    uid = Engine.comm_unique_id()
    errors = []
    threads = [threading.Thread(target=rank_main, args=(r, world, uid, all_datas, schema, errors)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise SystemExit(f"failed: {errors}")
    print(f"world {world}: ok")


if __name__ == "__main__":
    main()
