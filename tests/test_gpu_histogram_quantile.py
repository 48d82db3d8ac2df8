"""Histogram quantiles per label group and step (`hg_scan_histogram_quantile`, `Engine.scan_histogram_quantile`):
histogram_quantile(q, sum by (..., le) (fn(x[r]))) over classic histograms whose every `le` bucket is a series of its own.

Every case is compared with tests/histogram_model.py (a literal transcription of the definition in include/horae_gpu.h over the C oracle's
deduplicated stream) bit for bit: group, t and forced_monotonic as integers, quantiles as f64 bit patterns, a NaN matching any NaN.  Cases
marked `device_only` are too large for the emulated build of the library."""
import ctypes as C
import math
import os

import numpy as np
import pyarrow as pa
import pytest

import histogram_model as hm
from histogram_model import bucket_quantiles, histogram_quantile
from range_function_model import ALL_FNS, INCREASE, LAST_OVER_TIME, NAMES, RATE
from test_gpu_range_aggregates import _handle, _inputs, _schema, _write
from test_gpu_range_functions import _engine, _same
from horaedb_b200 import sstgen
from horaedb_b200._ffi import (HG_AGG_HASH, HG_AGG_RUNS, ArrowArrayStream, Engine, HgAggSpec, HgRangeSpec, SchemaHandle, _group_map, _make_preds,
                               _quantile_args)
from horaedb_b200.config import ParquetCompression, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode

pytestmark = pytest.mark.gpu
device_only = pytest.mark.skipif("HORAE_EMU_ORDER" in os.environ, reason="too large for the emulated library")
T0 = sstgen.T0_MS
U32_MAX = (1 << 32) - 1
INF = float("inf")
NAN = float("nan")
QS = (0.9, 0.0, 0.5, 1.0, 0.25, 0.99)          # shuffled on purpose
INT_COLS = ("group", "t", "forced_monotonic")


def _family(rng, n_groups, bounds, points, t0=T0, step=1000, key_lo=0, reset_p=0.05, jitter=True, dup=1):
    """Classic histograms: per group, one cumulative counter series per (bound, copy), all restarting together.  Observations fall into
    the buckets at random, so each bound's counter counts those at or below it; a series' samples are jittered on their own, so rates of
    one group's buckets are not monotonic in every window.  Returns the columns and the map (keys, groups, bounds)."""
    cols = {"series_id": [], "ts": [], "value": [], "tag": []}
    keys, groups, ubs = [], [], []
    sid = key_lo
    for g in range(n_groups):
        nb = len(bounds)
        obs = np.zeros(nb)
        traces = []
        for p in range(points):
            if rng.random() < reset_p:
                obs[:] = 0.0
            obs += rng.integers(0, 6, nb).astype(np.float64)
            traces.append(np.cumsum(obs))
        for b in range(nb):
            for _ in range(dup):
                for p in range(points):
                    cols["series_id"].append(sid)
                    cols["ts"].append(t0 + p * step + (int(rng.integers(0, step)) if jitter else 0))
                    cols["value"].append(float(traces[p][b]))
                    cols["tag"].append(int(rng.integers(0, 4)))
                keys.append(sid)
                groups.append(g)
                ubs.append(bounds[b])
                sid += 1
    return cols, (np.array(keys, np.uint64), np.array(groups, np.uint32), np.array(ubs, np.float64))


def _check(schema, datas, grid, maps, fns=(RATE,), qs=QS, preds=(), inputs=((0, False),), modes=(HG_AGG_RUNS,)):
    """every fn's table == the model's for each (keys, groups, bounds) in maps, for the given (flags, resident) inputs and modes; returns
    {(fn, j): the model's table}"""
    start, end, step, rng_ = grid
    handle = _handle(schema)
    exps = {(fn, j): histogram_quantile(datas, schema.arrow_schema, 2, fn, *m, qs, preds, start, end, step, rng_)
            for fn in fns for j, m in enumerate(maps)}
    for flags, resident in inputs:
        eng, ins = _engine(schema, datas, flags, resident)
        for mode in modes:
            for fn in fns:
                for j, (keys, groups, bounds) in enumerate(maps):
                    got = eng.scan_histogram_quantile(handle, ins, fn, keys, groups, bounds, qs, preds, start, end, step, rng_, mode=mode)
                    st = eng.stats()
                    _same(got, exps[(fn, j)], INT_COLS)
                    assert st["path"] == 0 and st["groups_out"] == got.num_rows, NAMES[fn]
                    assert st["bytes_d2h"] == got.num_rows * (4 + 8 + 1 + 8 * len(qs))
        eng.close()
    return exps


def _steps_reset():
    hm.STEPS.clear()


# ------------------------------------------------------------------------------------------------------------------------- grids
@pytest.mark.parametrize("step,rng_", [(5_000, 2_000),        # range < step
                                       (5_000, 5_000),        # range == step
                                       (3_000, 7_777),        # range > step, not a multiple of it
                                       (0, 10_000)],          # an instant query
                         ids=str)
def test_histogram_quantile_grids(step, rng_):
    rng = np.random.default_rng(step + rng_ + 3)
    schema = _schema()
    bounds = [0.05, 0.1, 0.5, 1.0, 5.0, INF]
    cols_a, map_a = _family(rng, 2, bounds, 40, key_lo=0)
    cols_b, map_b = _family(rng, 2, bounds, 40, key_lo=100)
    datas = [_write(schema, cols_a, 3, WriteConfig(max_row_group_size=200, compression=ParquetCompression.Snappy)),
             _write(schema, cols_b, 4, WriteConfig(max_row_group_size=200, compression=ParquetCompression.Uncompressed))]
    keys = np.concatenate([map_a[0], map_b[0]])
    groups = np.concatenate([map_a[1], map_b[1] + 2])
    ubs = np.concatenate([map_a[2], map_b[2]])
    grid = (T0 + 20_000, T0 + 20_000, step, rng_) if step == 0 else (T0 - 4_000, T0 + 45_000, step, rng_)
    exps = _check(schema, datas, grid, [(keys, groups, ubs)], fns=(RATE, INCREASE), modes=(HG_AGG_RUNS, HG_AGG_HASH),
                  inputs=((0, False), (0, True)))
    assert exps[(RATE, 0)].num_rows > 0 and set(exps[(RATE, 0)]["group"].to_pylist()) == {0, 1, 2, 3}


def test_histogram_quantile_every_function():
    rng = np.random.default_rng(61)
    schema = _schema()
    cols, m = _family(rng, 3, [0.25, 1.0, 4.0, INF], 30, reset_p=0.1)
    datas = [_write(schema, cols, 61)]
    exps = _check(schema, datas, (T0 + 2_000, T0 + 30_000, 2_500, 6_000), [m], fns=ALL_FNS)
    assert all(exps[(fn, 0)].num_rows > 0 for fn in ALL_FNS)


# ------------------------------------------------------------------------------------------------------------ the definition
def _explicit(series, t=T0 + 1_000):
    """one sample per series at t: series = [(key, value)]"""
    cols = {"series_id": [k for k, _ in series], "ts": [t] * len(series), "value": [v for _, v in series], "tag": [0] * len(series)}
    return cols


def _buckets_table(groups_buckets, key_lo=1):
    """groups_buckets = [(caller ordinal, [(bound, value), ...])]: one series per bucket; returns (cols, map)"""
    series, keys, groups, ubs = [], [], [], []
    k = key_lo
    for g, buckets in groups_buckets:
        for u, v in buckets:
            series.append((k, v))
            keys.append(k)
            groups.append(g)
            ubs.append(u)
            k += 1
    order = np.argsort(np.array([s[0] for s in series]))
    series = [series[i] for i in order]
    return _explicit(series), (np.array(keys, np.uint64), np.array(groups, np.uint32), np.array(ubs, np.float64))


INSTANT = (T0 + 1_000, T0 + 1_000, 0, 5_000)


def test_histogram_quantile_every_branch():
    """one (group, t) per branch of the definition, the model's counters asserting that each is reached"""
    up = math.nextafter(3.0, INF)
    cases = [(0, [(1.0, 5.0), (2.0, 7.0)]),                                   # no +inf bucket
             (1, [(INF, 5.0)]),                                               # the +inf bucket alone
             (2, [(1.0, 0.0), (INF, 0.0)]),                                   # obs == 0
             (3, [(0.1, 10.0), (0.2, 20.0), (INF, 40.0)]),                    # interpolation in the first / a later bucket, b = n - 1
             (4, [(-1.0, 10.0), (2.0, 18.0), (INF, 20.0)]),                   # b = 0 with u_0 <= 0
             (5, [(1.0, 10.0), (2.0, 8.0), (INF, 12.0)]),                     # forced monotonic
             (6, [(1.0, 3.0), (2.0, up), (INF, up)]),                         # the small-delta rule
             (7, [(1.0, NAN), (2.0, 5.0), (INF, 10.0)]),                      # a NaN sample in a count
             (8, [(-0.0, 3.0), (0.0, 4.0), (1.0, 8.0), (INF, 10.0)]),         # -0.0 and +0.0: one bucket
             (9, [(1.0, 2.0), (1.0, 3.0), (2.0, 6.0), (INF, 10.0)]),          # two series of one (group, bound): summed
             (10, [(-INF, 1.0), (-2.0, 3.0), (5.0, 6.0), (INF, 8.0)]),        # -inf and negative bounds
             (11, [(INF, 4.0), (1.0, 1.0), (3.0, 2.5)]),                      # buckets given out of bound order
             (U32_MAX, [(0.5, 1.0), (INF, 2.0)])]
    cols, m = _buckets_table(cases)
    schema = _schema()
    datas = [_write(schema, cols, 62)]
    qs = (0.0, 0.1, 0.25, 0.5, 0.9, 1.0)
    _steps_reset()
    exps = _check(schema, datas, INSTANT, [m], fns=(LAST_OVER_TIME,), qs=qs, modes=(HG_AGG_RUNS, HG_AGG_HASH))
    for step in ("no_inf", "inf_alone", "obs_zero", "b_last", "b0_nonpositive", "interp_first", "interp_later", "fixup_forced",
                 "fixup_small_delta"):
        assert hm.STEPS[step] > 0, step
    rows = {r["group"]: r for r in exps[(LAST_OVER_TIME, 0)].to_pylist()}
    assert sorted(rows) == [g for g, _ in cases]
    assert rows[5]["forced_monotonic"] == 1 and sum(r["forced_monotonic"] for r in rows.values()) == 1
    assert math.copysign(1.0, rows[8]["quantile_1"]) == 1.0 and rows[8]["quantile_1"] == 0.0   # one bucket 0.0 (+0.0) of count 7
    assert rows[10]["quantile_1"] == -INF


def test_histogram_quantile_worked_values():
    """the worked values of the definition, each written directly as one series per bucket and read with last_over_time"""
    up = math.nextafter(3.0, INF)
    cases = [  # (buckets, q, result, forced_monotonic)
        ([(0.1, 10.0), (0.2, 20.0), (INF, 40.0)], 0.1, 0.04000000000000001, 0),
        ([(0.1, 10.0), (0.2, 20.0), (INF, 40.0)], 0.25, 0.1, 0),
        ([(0.1, 10.0), (0.2, 20.0), (INF, 40.0)], 0.5, 0.2, 0),
        ([(0.1, 10.0), (0.2, 20.0), (INF, 40.0)], 0.9, 0.2, 0),
        ([(0.1, 10.0), (0.2, 20.0), (INF, 40.0)], 0.0, 0.0, 0),
        ([(1.0, 10.0), (2.0, 8.0), (INF, 12.0)], 0.5, 0.6, 1),
        ([(-1.0, 10.0), (2.0, 18.0), (INF, 20.0)], 0.5, -1.0, 0),
        ([(1.0, 3.0), (2.0, up), (INF, up)], 1.0, 1.0, 0),
        ([(1.0, 0.0), (INF, 0.0)], 0.5, NAN, 0),
        ([(INF, 5.0)], 0.5, NAN, 0),
        ([(1.0, 5.0), (2.0, 7.0)], 0.5, NAN, 0),
    ]
    schema = _schema()
    handle = _handle(schema)
    eng = Engine(device=0)
    for i, (buckets, q, want, flag) in enumerate(cases):
        cols, m = _buckets_table([(7, buckets)])
        ins = _inputs([_write(schema, cols, 70 + i)])
        got = eng.scan_histogram_quantile(handle, ins, LAST_OVER_TIME, *m, [q], [], *INSTANT).to_pylist()
        assert len(got) == 1 and got[0]["group"] == 7 and got[0]["t"] == INSTANT[0], i
        assert got[0]["forced_monotonic"] == flag, i
        v = got[0]["quantile_0"]
        assert (math.isnan(v) and math.isnan(want)) or (v == want and math.copysign(1, v) == math.copysign(1, want)), (i, v, want)
        mf, mv = bucket_quantiles(sorted(buckets), [q])                     # the model agrees with the worked value
        assert mf == flag and (mv[0] == want or (math.isnan(mv[0]) and math.isnan(want)))
    eng.close()


# -------------------------------------------------------------------------------------------------------------- relation, maps
def test_histogram_quantile_counts_are_the_by_map_sums():
    """the bucket counts are hg_scan_range_function_by_map's sums with the (group, bound) pair as the ordinal: bucketQuantile of those sums
    is the call's result bit for bit, the call's rows are the by-map rows' (group, t) projected on the group, and the dense tables are what
    bytes_h2d adds"""
    rng = np.random.default_rng(63)
    schema = _schema()
    bounds = [0.1, 0.3, 1.0, 3.0, INF]
    cols, (keys, groups, ubs) = _family(rng, 4, bounds, 40, dup=2, reset_p=0.1)
    groups = groups * 5 + 1                                                   # caller ordinals 1, 6, 11, 16
    datas = [_write(schema, cols, 63, WriteConfig(max_row_group_size=150))]
    grid = (T0 + 3_000, T0 + 40_000, 3_000, 9_000)
    handle = _handle(schema)
    eng, ins = _engine(schema, datas, 0, True)
    bidx = np.searchsorted(np.array(bounds), ubs)
    pair_ord = (groups // 5) * len(bounds) + bidx
    for fn in (RATE, INCREASE):
        sums = eng.scan_range_function_by_map(handle, ins, fn, keys, pair_ord, [], *grid)
        h_by_map = eng.stats()["bytes_h2d"]
        got = eng.scan_histogram_quantile(handle, ins, fn, keys, groups, ubs, QS, [], *grid)
        h_hist = eng.stats()["bytes_h2d"]
        cells = {}
        for r in sums.to_pylist():
            g = int(r["group"]) // len(bounds) * 5 + 1
            cells.setdefault((g, r["t"]), []).append((bounds[r["group"] % len(bounds)], r["sum"]))
        exp = [(g, t, *bucket_quantiles(cells[(g, t)], QS)) for g, t in sorted(cells)]
        _same(got, hm.histogram_table(exp, len(QS)), INT_COLS)
        assert got.num_rows > 0
        n_pairs, n_bounds, n_groups = len(set(zip(groups.tolist(), ubs.tolist()))), len(bounds), len(set(groups.tolist()))
        assert h_hist - h_by_map == 8 * n_pairs + 8 * n_bounds + 4 * n_groups
    eng.close()


def test_histogram_quantile_maps():
    """an empty map; series of the data missing from the map; map keys absent from the data; unsorted keys with repeats of one pair;
    caller ordinals 0 and 2^32 - 1"""
    rng = np.random.default_rng(64)
    schema = _schema()
    bounds = [0.5, 1.0, 2.0, INF]
    cols, (keys, groups, ubs) = _family(rng, 3, bounds, 30, key_lo=10)
    datas = [_write(schema, cols, 64, WriteConfig(max_row_group_size=100))]
    grid = (T0, T0 + 30_000, 2_000, 5_000)
    handle = _handle(schema)
    eng, ins = _engine(schema, datas)
    got = eng.scan_histogram_quantile(handle, ins, RATE, np.zeros(0, np.uint64), np.zeros(0, np.uint32), np.zeros(0), QS, [], *grid)
    assert got.num_rows == 0 and got.column_names == ["group", "t", "forced_monotonic"] + ["quantile_%d" % j for j in range(len(QS))]
    eng.close()
    groups = np.where(groups == 2, U32_MAX, groups).astype(np.uint32)
    keep = np.array([i for i in range(len(keys)) if i % 7 != 3])              # some series of the data are not in the map
    perm = rng.permutation(len(keep))
    k = np.concatenate([keys[keep][perm], keys[keep][:5], np.array([1, 2, 999_999], np.uint64)])
    g = np.concatenate([groups[keep][perm], groups[keep][:5], np.array([0, 5, 5], np.uint32)])
    b = np.concatenate([ubs[keep][perm], ubs[keep][:5], np.array([INF, 1.0, INF])])
    exps = _check(schema, datas, grid, [(k, g, b)], modes=(HG_AGG_RUNS, HG_AGG_HASH), inputs=((0, False), (0, True)))
    assert set(exps[(RATE, 0)]["group"].to_pylist()) == {0, 1, U32_MAX}


def test_histogram_quantile_long_segment():
    """300 bounds in one group (a segment of 300 buckets for one thread)"""
    rng = np.random.default_rng(65)
    schema = _schema()
    bounds = [float(i) * 0.25 - 10.0 for i in range(299)] + [INF]
    cols, m = _family(rng, 1, bounds, 6, step=2_000)
    datas = [_write(schema, cols, 65, WriteConfig(max_row_group_size=1000))]
    exps = _check(schema, datas, (T0 + 4_000, T0 + 12_000, 4_000, 6_000), [m], fns=(RATE, LAST_OVER_TIME))
    assert exps[(RATE, 0)].num_rows > 0


@device_only
def test_histogram_quantile_many_series():
    """2 004 series (167 groups x 12 bounds) over 300 steps"""
    rng = np.random.default_rng(66)
    schema = _schema()
    bounds = [0.005, 0.01, 0.025, 0.05, 0.1, 0.25, 0.5, 1.0, 2.5, 5.0, 10.0, INF]
    cols, m = _family(rng, 167, bounds, 40, step=10_000, reset_p=0.02)
    datas = [_write(schema, cols, 66, WriteConfig(max_row_group_size=8192))]
    exps = _check(schema, datas, (T0 + 30_000, T0 + 30_000 + 299 * 1_300, 1_300, 30_000), [m], fns=(RATE,))
    assert exps[(RATE, 0)].num_rows > 100 * 167


# ------------------------------------------------------------------------------------------------------- refusals, empty results
def _raw(eng, handle, ins, spec, grid, fn, m, bounds, qs, nq=None, preds=()):
    arr, keep = eng._descs(ins)
    p = _make_preds(handle.arrow_schema, preds)
    stream = ArrowArrayStream()
    qarr, qn = _quantile_args(qs)
    if bounds is None:
        b = None
    else:
        b = np.ascontiguousarray(bounds, dtype=np.float64)
        keep = (keep, b)
        b = C.cast(C.c_void_p(b.ctypes.data), C.POINTER(C.c_double))
    return eng._L.hg_scan_histogram_quantile(eng._h, C.byref(handle.desc), arr, C.c_size_t(len(ins)), p, C.c_size_t(len(preds)), C.byref(spec),
                                             C.byref(HgRangeSpec(*grid)), C.c_uint32(fn), C.byref(m), b, qarr,
                                             qn if nq is None else C.c_uint32(nq), C.byref(stream))


def test_histogram_quantile_refusals_before_device_work():
    rng = np.random.default_rng(67)
    schema = _schema()
    cols, (keys, groups, ubs) = _family(rng, 2, [1.0, INF], 10)
    handle = _handle(schema)
    ins = _inputs([_write(schema, cols, 67)])
    good = (T0, T0 + 10_000, 1_000, 5_000)
    m = _group_map(schema.arrow_schema, 0, keys, groups)
    kb = ubs.tolist()
    conflict = _group_map(schema.arrow_schema, 0, [1, 2, 1], [0, 0, 0])
    append = StorageSchema.try_new(pa.schema([pa.field("series_id", pa.uint64()), pa.field("ts", pa.int64()), pa.field("blob", pa.binary())]), 2,
                                   UpdateMode.Append)
    handle_a = SchemaHandle(append.arrow_schema, 2, UpdateMode.Append)
    # 2^21 distinct groups over 2^20 distinct bounds with 2^24 steps: 21 + 24 + 20 = 65 key bits
    nw = 1 << 21
    wide = _group_map(schema.arrow_schema, 0, np.arange(nw, dtype=np.uint64), np.arange(nw, dtype=np.uint32))
    wide_b = (np.arange(nw) % (1 << 20)).astype(np.float64)
    wide_grid = (0, (1 << 24) - 1, 1, 5)
    eng = Engine(device=0)
    eng.scan_histogram_quantile(handle, ins, RATE, keys, groups, ubs, QS, [], *good)
    before = eng.stats()
    assert before["kernel_launches"] > 0
    spec = HgAggSpec(0, 1, 0, 2, 0)
    cases = [  # (handle, inputs, spec, grid, fn, map, bounds, qs, n_quantiles, preds, code, message)
        (handle, ins, spec, good, RATE, m, [kb[0], NAN] + kb[2:], (0.5,), None, (), 1, "histogram map: a NaN upper bound"),     # a NaN bound
        (handle, ins, spec, good, RATE, conflict, [1.0, INF, 2.0], (0.5,), None, (), 1, "group map: a key mapped to two different groups"),  # key 1 with two bounds
        (handle, ins, spec, good, RATE, _group_map(schema.arrow_schema, 0, [1, 2, 1], [0, 0, 1]), [1.0, INF, 1.0], (0.5,), None, (), 1, "group map: a key mapped to two different groups"),
        (handle, ins, spec, good, RATE, m, None, (0.5,), None, (), 1, "histogram map: null upper bounds"),                      # null bounds
        (handle, ins, spec, good, RATE, m, kb, (1.5,), None, (), 1, "a quantile must lie in [0, 1]"),                           # q outside [0, 1]
        (handle, ins, spec, good, RATE, m, kb, (-0.1,), None, (), 1, "a quantile must lie in [0, 1]"),
        (handle, ins, spec, good, RATE, m, kb, (NAN,), None, (), 1, "a quantile must lie in [0, 1]"),
        (handle, ins, spec, good, RATE, m, kb, (0.5,), 0, (), 1, "a quantile aggregate takes 1 to 16 quantiles"),               # 0 quantiles
        (handle, ins, spec, good, RATE, m, kb, (0.5,) * 17, None, (), 1, "a quantile aggregate takes 1 to 16 quantiles"),       # 17 quantiles
        (handle, ins, spec, good, LAST_OVER_TIME + 1, m, kb, (0.5,), None, (), 1, "range function: fn is not an hg_range_fn"),  # fn outside the enum
        (handle, ins, spec, good, RATE, m, kb, (0.5,), None, [("tag", "ge", 0)] * 6, 2, "more than 5 predicates (the map's set and the range's time bounds take three of 8)"),  # 6 caller predicates
        (handle_a, [], HgAggSpec(0, 1, 0, 1, 0), good, RATE, m, kb, (0.5,), None, (), 2, "aggregation over an Append-mode (BytesMergeOperator) table"),  # an Append-mode table, without any SST
        (handle, ins, HgAggSpec(0, 1, 1000, 2, 0), good, RATE, m, kb, (0.5,), None, (), 1, "a range aggregate takes its windows from the range spec: window_ms must be <= 0"),  # window_ms > 0
        (handle, ins, spec, wide_grid, RATE, wide, wide_b, (0.5,), None, (), 2, "histogram quantile: the sort key (group, step, bound) needs more than 64 bits"),  # a sort key of 65 bits
        (handle, ins, spec, good, RATE, m, [kb[0], NAN] + kb[2:], (1.5,), None, (), 1, "a quantile must lie in [0, 1]"),        # two faults: the quantiles before the bounds
        (handle, ins, spec, (T0 + 10, T0, 1_000, 5_000), RATE, m, kb, (1.5,), None, (), 1, "range spec: start_ms > end_ms"),    # and the range before the quantiles
    ]
    for h, ii, sp, grid, fn, mm, b, qs, nq, preds, code, message in cases:
        rc = _raw(eng, h, ii, sp, grid, fn, mm, b, qs, nq, preds)
        assert rc == code, (grid, fn, b if b is None or len(b) < 8 else len(b), qs, nq, len(preds), rc, eng._L.hg_last_error())
        assert eng._L.hg_last_error().decode() == message, (rc, eng._L.hg_last_error())
        assert eng.stats() == before, (grid, fn, qs)
    # 5 caller predicates are accepted
    assert _raw(eng, handle, ins, spec, (T0, T0 + 10_000, 1_000, 5_000), RATE, m, kb, QS[:5], None, [("tag", "ge", 0)] * 5) == 0
    eng.close()


def test_histogram_quantile_empty_input_and_no_passing_row():
    schema = _schema()
    rng = np.random.default_rng(68)
    cols, m = _family(rng, 2, [1.0, INF], 10)
    data = _write(schema, cols, 68)
    h = _handle(schema)
    names = ["group", "t", "forced_monotonic", "quantile_0", "quantile_1"]
    for datas, preds in (([], []), ([data], [("tag", "gt", 10)])):
        eng, ins = _engine(schema, datas)
        got = eng.scan_histogram_quantile(h, ins, RATE, *m, (0.5, 0.9), preds, T0, T0 + 60_000, 1_000, 5_000)
        assert got.num_rows == 0 and got.column_names == names
        assert got.schema.field("forced_monotonic").type == pa.uint8() and got.schema.field("group").type == pa.uint32()
        st = eng.stats()
        assert st["groups_out"] == 0 and st["bytes_d2h"] == 0 and st["path"] == 0
        eng.close()
