"""Top-k and bottom-k series per label group and step (`hg_scan_range_function_topk`, `Engine.scan_range_function_topk`): the windows
and values of `hg_scan_range_function_by_map`, ranked per (group, t) by value (NaN last, ties in series-key order) and cut to k.

Every case is compared with tests/topk_model.py (a literal transcription of the definition in include/horae_gpu.h over the C oracle's
deduplicated stream) bit for bit: groups, times and keys as integers, values as f64 bit patterns (-0.0 is not +0.0), any NaN matching any
NaN.  Cases marked `device_only` are too large for the emulated build of the library."""
import ctypes as C
import math
import os

import numpy as np
import pyarrow as pa
import pytest

from range_function_model import ALL_FNS, CHANGES, COUNT_OVER_TIME, IRATE, LAST_OVER_TIME, MAX_OVER_TIME, NAMES, RATE, RESETS, SUM_OVER_TIME
from test_gpu_range_aggregates import _cols, _f64_bits, _handle, _inputs, _schema, _write
from test_gpu_range_functions import _engine, _same, _spread_map
from topk_model import range_function_topk
from horaedb_b200 import sstgen
from horaedb_b200._ffi import (HG_AGG_HASH, HG_AGG_RUNS, HG_BOTTOMK, HG_FLAG_NO_PRUNING, HG_TOPK, ArrowArrayStream, Engine, HgAggSpec, HgRangeSpec,
                               SchemaHandle, _group_map, _make_preds)
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode

pytestmark = pytest.mark.gpu
device_only = pytest.mark.skipif("HORAE_EMU_ORDER" in os.environ, reason="too large for the emulated library")
T0 = sstgen.T0_MS
U32_MAX = (1 << 32) - 1
ORDERS = (HG_TOPK, HG_BOTTOMK)


def _check(schema, datas, grid, maps, fns=(RATE,), ks=(1, 3, 1000), orders=ORDERS, preds=(), oracle_preds=None, inputs=((0, False),),
           modes=(HG_AGG_RUNS,), model=None):
    """the call's table == the model's for every (fn, k, order, map) and (flags, resident) input and mode, with its stats; returns
    {(fn, k, order, map index): the model's table}"""
    start, end, step, rng_ = grid
    op = oracle_preds if oracle_preds is not None else preds
    npk = getattr(schema, "npk", 2)
    handle = _handle(schema)
    ms, md = model or (schema, datas)
    key_name = schema.arrow_schema.field(0).name
    kw = schema.arrow_schema.field(0).type.bit_width // 8
    exps = {(fn, k, o, j): range_function_topk(md, ms.arrow_schema, npk, fn, k, keys, groups, o, op, start, end, step, rng_)
            for fn in fns for k in ks for o in orders for j, (keys, groups) in enumerate(maps)}
    for flags, resident in inputs:
        eng, ins = _engine(schema, datas, flags, resident)
        for mode in modes:
            for (fn, k, o, j), exp in exps.items():
                keys, groups = maps[j]
                got = eng.scan_range_function_topk(handle, ins, fn, k, keys, groups, preds, start, end, step, rng_, order=o, mode=mode)
                st = eng.stats()
                _same(got, exp, ("group", "t", key_name))
                assert st["path"] == 0 and st["groups_out"] == got.num_rows, (NAMES[fn], k, o)
                assert st["bytes_d2h"] == got.num_rows * (4 + 8 + kw + 8)
        eng.close()
    return exps


def _series_rows(sids_vals, t_step=1000):
    cols = {"series_id": [], "ts": [], "value": [], "tag": []}
    for sid, vals in sids_vals:
        for i, v in enumerate(vals):
            cols["series_id"].append(sid)
            cols["ts"].append(T0 + t_step * i)
            cols["value"].append(v)
            cols["tag"].append(0)
    return cols


# ------------------------------------------------------------------------------------------------------------------------- grids
@pytest.mark.parametrize("step,rng_", [(5_000, 2_000),        # range < step
                                       (5_000, 5_000),        # range == step
                                       (3_000, 7_777),        # range > step, not a multiple of it
                                       (0, 10_000)],          # an instant query
                         ids=str)
def test_range_topk_grids(step, rng_):
    rng = np.random.default_rng(step + rng_ + 3)
    schema = _schema()
    cols = _cols(rng, 9, 50, reset_p=0.1, null_p=0.05)
    grid = (T0 + 20_000, T0 + 20_000, step, rng_) if step == 0 else (T0 - 4_000, T0 + 60_000, step, rng_)
    exps = _check(schema, [_write(schema, cols, 3)], grid, [_spread_map(9, 2)], ks=(1, 3, 9), modes=(HG_AGG_RUNS, HG_AGG_HASH),
                  inputs=((0, False), (0, True)))
    assert all(e.num_rows > 0 for e in exps.values())
    # k = 3 cuts some (group, t): a group holds 4 or 5 series
    assert exps[(RATE, 3, HG_TOPK, 0)].num_rows < exps[(RATE, 9, HG_TOPK, 0)].num_rows


def test_range_topk_every_function():
    rng = np.random.default_rng(61)
    schema = _schema()
    cols = _cols(rng, 7, 40, reset_p=0.15, null_p=0.05)
    _check(schema, [_write(schema, cols, 61)], (T0, T0 + 40_000, 2_500, 6_000), [_spread_map(7, 3)], fns=ALL_FNS, ks=(2,))


# -------------------------------------------------------------------------------------------------------------- ties and specials
def test_range_topk_ties_decided_by_series_key():
    """count_over_time and resets give many equal values: the series key decides among them, in both directions; -0.0 and +0.0 are
    equal values reported with their own bits"""
    rng = np.random.default_rng(63)
    schema = _schema()
    cols = _cols(rng, 12, 30, step=1000, reset_p=0.3, jitter=False)
    datas = [_write(schema, cols, 63)]
    keys = np.arange(12, dtype=np.uint64)[::-1].copy()                           # an unsorted map
    groups = (np.arange(12)[::-1] % 2).astype(np.uint32)
    exps = _check(schema, datas, (T0 + 5_000, T0 + 29_000, 3_000, 5_000), [(keys, groups)], fns=(COUNT_OVER_TIME, RESETS), ks=(1, 4))
    exp = exps[(COUNT_OVER_TIME, 4, HG_TOPK, 0)]
    by = {}
    for g, t, s in zip(exp["group"].to_pylist(), exp["t"].to_pylist(), exp["series_id"].to_pylist()):
        by.setdefault((g, t), []).append(s)
    assert any(v == sorted(v) and len(v) == 4 for v in by.values())            # all equal counts: the first four series keys
    zeros = _series_rows([(1, [0.0, -0.0, -0.0]), (2, [0.0, 0.0, 0.0]), (3, [-0.0, 0.0, -0.0]), (4, [1.0, -1.0, 0.0])])
    zdatas = [_write(schema, zeros, 64)]
    exps = _check(schema, zdatas, (T0, T0 + 2_000, 1_000, 1_000), [(np.arange(1, 5, dtype=np.uint64), np.zeros(4, np.uint32))],
                  fns=(LAST_OVER_TIME,), ks=(1, 2, 4))
    bits = _f64_bits(exps[(LAST_OVER_TIME, 4, HG_BOTTOMK, 0)]["value"].combine_chunks())
    assert 0x8000000000000000 in bits and 0 in bits


def test_range_topk_nan_and_infinities():
    """NaN after every other value in both directions, NaNs in series order when fewer than k values are not NaN; ±inf ranked as values"""
    schema = _schema()
    inf, nan = float("inf"), float("nan")
    rows = [(1, [nan, nan, 1.0, nan]), (2, [1.0, -nan, nan, -inf]), (3, [-inf, 2.0, nan, inf]), (4, [nan, inf, -1.0, nan]),
            (5, [3.0, nan, nan, nan]), (6, [None, -inf, nan, 0.5])]
    datas = [_write(schema, _series_rows(rows), 65)]
    exps = _check(schema, datas, (T0, T0 + 3_000, 1_000, 1_000), [(np.arange(1, 7, dtype=np.uint64), np.zeros(6, np.uint32))],
                  fns=(LAST_OVER_TIME,), ks=(1, 2, 3, 6))
    for o in ORDERS:
        exp = exps[(LAST_OVER_TIME, 6, o, 0)]
        for t in set(exp["t"].to_pylist()):
            vs = [v for tt, v in zip(exp["t"].to_pylist(), exp["value"].to_pylist()) if tt == t]
            nans = [math.isnan(v) for v in vs]
            assert nans == sorted(nans)                                           # NaN last
    exp = exps[(LAST_OVER_TIME, 3, HG_TOPK, 0)]
    at2 = [(s, v) for t, s, v in zip(exp["t"].to_pylist(), exp["series_id"].to_pylist(), exp["value"].to_pylist()) if t == T0 + 2_000]
    assert [s for s, _ in at2] == [1, 4, 2]                                       # 1.0, -1.0, then the first NaN in series order


# ------------------------------------------------------------------------------------------------------------ the by-map relation
def test_range_topk_against_the_by_map_call():
    """rows per (group, t) = min(k, count); k = 1 is the by-map max (HG_TOPK) / min (HG_BOTTOMK) bit for bit where no value is NaN; the
    map's upload counts as the by-map call's"""
    rng = np.random.default_rng(67)
    schema = _schema()
    cols = _cols(rng, 10, 40, reset_p=0.1, null_p=0.05)
    datas = [_write(schema, cols, 67)]
    grid = (T0, T0 + 40_000, 2_000, 5_000)
    keys, groups = _spread_map(10, 3)
    eng, ins = _engine(schema, datas)
    h = _handle(schema)
    for fn in (RATE, IRATE, SUM_OVER_TIME):
        bm = eng.scan_range_function_by_map(h, ins, fn, keys, groups, [], *grid)
        h2d = eng.stats()["bytes_h2d"]
        count = {(g, t): c for g, t, c in zip(bm["group"].to_pylist(), bm["t"].to_pylist(), bm["count"].to_pylist())}
        for k in (1, 2, 5):
            for o in ORDERS:
                got = eng.scan_range_function_topk(h, ins, fn, k, keys, groups, [], *grid, order=o)
                assert eng.stats()["bytes_h2d"] == h2d
                n = {}
                for g, t in zip(got["group"].to_pylist(), got["t"].to_pylist()):
                    n[(g, t)] = n.get((g, t), 0) + 1
                assert n == {gt: min(k, c) for gt, c in count.items()}, (NAMES[fn], k, o)
                if k == 1:
                    col = "max" if o == HG_TOPK else "min"
                    want = [_f64_bits(pa.array([v]))[0] for v in bm[col].to_pylist()]
                    have = _f64_bits(got["value"].combine_chunks())
                    assert len(have) == len(want) and all(a == b for a, b, v in zip(have, want, bm[col].to_pylist()) if not math.isnan(v))
    eng.close()


# ------------------------------------------------------------------------------------------------------------------------- maps
def test_range_topk_maps():
    """series outside the map are absent; an empty map gives an empty result; ordinals up to 2^32 - 1; one global group; one group per
    series (every series is its own top-1)"""
    rng = np.random.default_rng(69)
    schema = _schema()
    cols = _cols(rng, 12, 30, key_lo=100, null_p=0.05, reset_p=0.1)
    datas = [_write(schema, cols, 69, WriteConfig(max_row_group_size=100))]
    grid = (T0, T0 + 30_000, 2_000, 4_000)
    keys = np.array([109, 100, 103, 104, 105, 101, 110, 100, 103, 111, 5, 7], np.uint64)
    groups = np.array([3, 0, 0, 0, 3, 3, 3, 0, 0, U32_MAX, 1, 1], np.uint32)   # 102, 106-108 are not in the map; 5, 7 are in no file
    every = np.arange(100, 112, dtype=np.uint64)
    maps = [(keys, groups), (every, np.zeros(12, np.uint32)), (every, np.arange(12, dtype=np.uint32)),
            (every, np.full(12, U32_MAX, np.uint32))]
    exps = _check(schema, datas, grid, maps, fns=(RATE, MAX_OVER_TIME), ks=(1, 2, 12), modes=(HG_AGG_RUNS, HG_AGG_HASH),
                  inputs=((0, False), (0, True)))
    e0 = exps[(RATE, 12, HG_TOPK, 0)]
    assert set(e0["group"].to_pylist()) == {0, 3, U32_MAX} and not set(e0["series_id"].to_pylist()) & {102, 106, 107, 108}
    e2 = exps[(RATE, 1, HG_TOPK, 2)]
    assert e2.num_rows == exps[(RATE, 12, HG_TOPK, 2)].num_rows
    eng, ins = _engine(schema, datas)
    got = eng.scan_range_function_topk(_handle(schema), ins, RATE, 3, np.zeros(0, np.uint64), np.zeros(0, np.uint32), [], *grid)
    assert got.num_rows == 0 and got.column_names == ["group", "t", "series_id", "value"]
    eng.close()


@device_only
def test_range_topk_many_series_and_steps():
    """2 000 series over 1 000+ steps in 7 groups, and one (group, t) segment of 100 000 series"""
    rng = np.random.default_rng(71)
    schema = _schema()
    cols = _cols(rng, 2000, 40, step=30_000, reset_p=0.02)
    datas = [_write(schema, cols, 71, WriteConfig(max_row_group_size=8192))]
    keys, groups = _spread_map(2000, 7)
    _check(schema, datas, (T0, T0 + 1_199_000, 1_000, 60_000), [(keys, groups)], ks=(1, 10, 400))
    n = 100_000
    big = {"series_id": list(range(n)), "ts": [T0] * n, "value": [float(rng.integers(0, 50)) for _ in range(n)], "tag": [0] * n}
    bdatas = [_write(schema, big, 72, WriteConfig(max_row_group_size=65536))]
    _check(schema, bdatas, (T0, T0, 0, 1_000), [(np.arange(n, dtype=np.uint64), np.zeros(n, np.uint32))], fns=(LAST_OVER_TIME,),
           ks=(1, 10, 99_999, 100_000))


# ------------------------------------------------------------------------------------------------------------------------- inputs
def test_range_topk_overwritten_rows_across_overlapping_ssts():
    rng = np.random.default_rng(73)
    schema = _schema()
    old = _cols(rng, 6, 40, jitter=False, reset_p=0.1)
    new = {k: v[::3] for k, v in old.items()}
    new["value"] = [v + 1000.0 if v is not None else None for v in new["value"]]
    datas = [_write(schema, old, 20), _write(schema, new, 21)]
    _check(schema, datas, (T0, T0 + 45_000, 4_000, 10_000), [_spread_map(6, 2)], fns=(RATE, SUM_OVER_TIME), ks=(1, 2),
           inputs=((0, False), (0, True), (HG_FLAG_NO_PRUNING, False)))


@pytest.mark.parametrize("codec", [ParquetCompression.Snappy, ParquetCompression.Zstd])
@pytest.mark.parametrize("kind", ["plain", "delta_dict"])
def test_range_topk_codecs_and_encodings(codec, kind):
    rng = np.random.default_rng(75)
    schema = _schema(value_t=pa.int64())
    cols = _cols(rng, 5, 50, ints=True, null_p=0.03)
    cols["value"] = [None if v is None else int(v) for v in cols["value"]]
    opts = {} if kind == "plain" else {"ts": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                       "series_id": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                       "value": ColumnOptions(enable_dict=True)}
    cfg = WriteConfig(compression=codec, max_row_group_size=100, column_options=opts)
    _check(schema, [_write(schema, cols, 22, cfg)], (T0 + 5_000, T0 + 50_000, 5_000, 15_000), [_spread_map(5, 2)], fns=(RATE, CHANGES),
           ks=(1, 3), inputs=((0, False), (0, True)))


def test_range_topk_integer_values_above_2_53_and_signed_keys():
    """u64 / i64 values near 2^63 and around 2^53 (rounded to f64 as the per-series call rounds them); an i64 series key with negative keys"""
    rng = np.random.default_rng(77)
    for key_t, value_t in ((pa.uint64(), pa.uint64()), (pa.int64(), pa.int64())):
        schema = _schema(key_t=key_t, value_t=value_t)
        cols = _cols(rng, 6, 20, key_lo=-3 if key_t == pa.int64() else 0)
        hi = (1 << 64) - 1 if value_t == pa.uint64() else (1 << 63) - 1
        edge = [hi, hi - 1, (1 << 53) - 1, 1 << 53, (1 << 53) + 1, (1 << 53) + 2]
        cols["value"] = [edge[(i * 7 + i // 20) % len(edge)] for i in range(len(cols["value"]))]
        keys = np.array(sorted(set(cols["series_id"])), np.int64)
        _check(schema, [_write(schema, cols, 78)], (T0, T0 + 20_000, 2_000, 3_000), [(keys, (np.arange(6) % 2).astype(np.uint32))],
               fns=(LAST_OVER_TIME, MAX_OVER_TIME), ks=(1, 3))


def test_range_topk_caller_predicates():
    """`tag = k` beside the map's set and the time bounds, and 5 caller predicates (the most the call accepts)"""
    rng = np.random.default_rng(79)
    schema = _schema()
    cols = _cols(rng, 12, 30, key_lo=1000, null_p=0.02)
    datas = [_write(schema, cols, 79, WriteConfig(max_row_group_size=200))]
    grid = (T0 + 3_000, T0 + 28_000, 2_500, 6_000)
    maps = [_spread_map(12, 3, key_lo=1000)]
    _check(schema, datas, grid, maps, ks=(1, 2), preds=[("tag", "eq", 2)])
    _check(schema, datas, grid, maps, ks=(2,), orders=(HG_BOTTOMK,), preds=[("tag", "ge", 0)] * 4 + [("series_id", "ne", 1003)])


# ------------------------------------------------------------------------------------------------------- refusals, empty results
def _raw(eng, handle, ins, spec, rs, fn, m, k, order, preds=()):
    arr, keep = eng._descs(ins)
    p = _make_preds(handle.arrow_schema, preds)
    stream = ArrowArrayStream()
    return eng._L.hg_scan_range_function_topk(eng._h, C.byref(handle.desc), arr, C.c_size_t(len(ins)), p, C.c_size_t(len(preds)),
                                              C.byref(spec), C.byref(rs) if rs is not None else None, C.c_uint32(fn),
                                              C.byref(m) if m is not None else None, C.c_uint32(k), C.c_uint32(order), C.byref(stream))


def test_range_topk_refusals_before_device_work():
    rng = np.random.default_rng(81)
    schema = _schema(extra=[pa.field("blob", pa.binary()), pa.field("fval", pa.float32())])
    cols = _cols(rng, 3, 10)
    cols["blob"] = [b"x"] * len(cols["ts"])
    cols["fval"] = [1.0] * len(cols["ts"])
    handle = _handle(schema)
    ins = _inputs([_write(schema, cols, 81)])
    good = (T0, T0 + 10_000, 1_000, 5_000)
    m = _group_map(schema.arrow_schema, 0, [0, 1, 2], [0, 0, 1])
    dup = _group_map(schema.arrow_schema, 0, [1, 0, 1], [0, 0, 1])
    append = StorageSchema.try_new(pa.schema([pa.field("series_id", pa.uint64()), pa.field("ts", pa.int64()), pa.field("blob", pa.binary())]), 2,
                                   UpdateMode.Append)
    handle_a = SchemaHandle(append.arrow_schema, 2, UpdateMode.Append)
    eng = Engine(device=0)
    eng.scan_range_function_topk(handle, ins, RATE, 2, [0, 1, 2], [0, 0, 1], [], *good)
    before = eng.stats()
    assert before["kernel_launches"] > 0
    cases = [  # (handle, inputs, spec kwargs, range spec, fn, map, k, order, preds, code, message)
        (handle, ins, {}, good, RATE, m, 0, HG_TOPK, (), 1, "top-k: k must be >= 1"),                                         # k = 0
        (handle, ins, {}, good, RATE, m, 1, 2, (), 1, "top-k: order is not an hg_topk_order"),                                # order outside the enum
        (handle, ins, {}, good, LAST_OVER_TIME + 1, m, 1, HG_TOPK, (), 1, "range function: fn is not an hg_range_fn"),        # fn outside the enum
        (handle, ins, {}, good, RATE, m, 1, HG_TOPK, [("tag", "ge", 0)] * 6, 2, "more than 5 predicates (the map's set and the range's time bounds take three of 8)"),  # 6 caller predicates (5 are accepted)
        (handle, ins, {}, None, RATE, m, 1, HG_TOPK, (), 1, "null range spec"),                                               # the range refusals
        (handle, ins, {}, (T0, T0 + 10, 0, 5), RATE, m, 1, HG_TOPK, (), 1, "range spec: step_ms must be > 0"),
        (handle, ins, {}, (T0 + 10, T0, 1, 5), RATE, m, 1, HG_BOTTOMK, (), 1, "range spec: start_ms > end_ms"),
        (handle, ins, {"window_ms": 1000}, good, RATE, m, 1, HG_TOPK, (), 1, "a range aggregate takes its windows from the range spec: window_ms must be <= 0"),
        (handle, ins, {"value_col": 4}, good, RATE, m, 1, HG_TOPK, (), 1, "Binary columns cannot be grouped or aggregated"),  # Binary value column
        (handle, ins, {"group_col": 3}, good, RATE, m, 1, HG_TOPK, (), 2, "counter aggregate: the group column must be the first primary key (one series per group)"),  # not one series per window
        (handle, ins, {"mode": 2}, good, RATE, m, 1, HG_TOPK, (), 1, "aggregation mode"),
        (handle, ins, {}, good, RATE, None, 1, HG_TOPK, (), 1, "null group map"),                                             # the map refusals
        (handle, ins, {}, good, RATE, dup, 1, HG_TOPK, (), 1, "group map: a key mapped to two different groups"),             # a key mapped to two groups
        (handle, ins, {"group_col": 5}, good, RATE, m, 1, HG_TOPK, (), 2, "counter aggregate: the group column must be the first primary key (one series per group)"),  # a float key column is not the series
        (handle_a, [], {"value_col": 1}, good, RATE, m, 1, HG_TOPK, (), 2, "aggregation over an Append-mode (BytesMergeOperator) table"),  # an Append-mode table, without any SST too
        (handle, ins, {}, good, RATE, dup, 0, HG_TOPK, (), 1, "top-k: k must be >= 1"),                                       # two faults: k is reported before the map's keys are read
        (handle, ins, {"value_col": 4}, good, RATE, m, 0, HG_TOPK, (), 1, "Binary columns cannot be grouped or aggregated"),  # and the spec before k
    ]
    for h, ii, kw, grid, fn, mm, k, order, preds, code, message in cases:
        spec = HgAggSpec(kw.get("group_col", 0), kw.get("ts_col", 1), kw.get("window_ms", 0), kw.get("value_col", 2), kw.get("mode", 0))
        rc = _raw(eng, h, ii, spec, HgRangeSpec(*grid) if grid is not None else None, fn, mm, k, order, preds)
        assert rc == code, (kw, grid, fn, k, order, len(preds), rc, eng._L.hg_last_error())
        assert eng._L.hg_last_error().decode() == message, (rc, eng._L.hg_last_error())
        assert eng.stats() == before, (kw, grid, fn, k, order)
    assert eng.scan_range_function_topk(handle, ins, RATE, 1, [0, 1, 2], [0, 0, 1], [("tag", "ge", 0)] * 5, *good).num_rows > 0
    assert eng.scan_range_function_topk(handle, ins, RATE, U32_MAX, [0, 1, 2], [0, 0, 1], [], *good, order=HG_BOTTOMK).num_rows > 0
    eng.close()


def test_range_topk_empty_input_and_no_passing_row():
    schema = _schema()
    rng = np.random.default_rng(83)
    data = _write(schema, _cols(rng, 3, 10), 83)
    h = _handle(schema)
    for datas, preds in (([], []), ([data], [("tag", "gt", 10)])):
        eng, ins = _engine(schema, datas)
        got = eng.scan_range_function_topk(h, ins, RATE, 2, [0, 1, 2], [0, 1, 1], preds, T0, T0 + 60_000, 1_000, 5_000)
        assert got.num_rows == 0 and got.column_names == ["group", "t", "series_id", "value"]
        st = eng.stats()
        assert st["groups_out"] == 0 and st["bytes_d2h"] == 0
        eng.close()
