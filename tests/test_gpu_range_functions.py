"""PromQL range functions (`hg_scan_range_function`, `hg_scan_range_function_by_map`, `Engine.scan_range_function` / `_by_map`): one
value per series and evaluation step (rate, increase, delta, irate, idelta, resets, changes, *_over_time), computed by
range_function_kernel over the range windows, and their count / sum / min / max across the series of a label group.

Every case is compared with tests/range_function_model.py (a literal transcription of the definitions in include/horae_gpu.h over the C
oracle's deduplicated stream) bit for bit: keys, times and counts as integers, values as f64 bit patterns.  NaN is the one exception: IEEE
leaves the payload of a NaN result to the hardware, so a NaN matches any NaN.  Cases marked `device_only` are too large for the emulated
build of the library."""
import ctypes as C
import os
from fractions import Fraction

import numpy as np
import pyarrow as pa
import pytest

from range_function_model import (ALL_FNS, CHANGES, COUNT_OVER_TIME, DELTA, IDELTA, INCREASE, IRATE, LAST_OVER_TIME, MAX_OVER_TIME, MIN_OVER_TIME,
                                  NAMES, RATE, RESETS, SUM_OVER_TIME, extrapolation, function_windows, range_function, range_function_by_map)
from range_model import _windows
from test_gpu_range_aggregates import _cols, _f64_bits, _handle, _inputs, _schema, _write
from horaedb_b200 import sstgen
from horaedb_b200._ffi import (HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_PRUNING, HG_FN_LAST_OVER_TIME, HG_FN_RATE, ArrowArrayStream, Engine, HgAggSpec,
                               HgRangeSpec, SchemaHandle, _group_map, _make_preds)
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode

pytestmark = pytest.mark.gpu
device_only = pytest.mark.skipif("HORAE_EMU_ORDER" in os.environ, reason="too large for the emulated library")
T0 = sstgen.T0_MS
U32_MAX = (1 << 32) - 1


def _same(got, exp, int_cols):
    assert got.column_names == exp.column_names
    assert got.num_rows == exp.num_rows, (got.num_rows, exp.num_rows)
    for i, name in enumerate(exp.column_names):
        g, e = got[name].combine_chunks(), exp[name].combine_chunks()
        assert g.type == e.type, (name, g.type, e.type)
        assert g.null_count == 0, name
        if name in int_cols:
            assert g.to_pylist() == e.to_pylist(), name
        else:
            assert _f64_bits(g) == _f64_bits(e), name


def _engine(schema, datas, flags=0, resident=False):
    eng = Engine(device=0, flags=flags)
    ins = _inputs(datas)
    if resident:
        h = _handle(schema)
        for i in range(len(ins)):
            eng.load_sst(h, ins[i])
            ins[i] = type(ins[i])(id=ins[i].id)
    return eng, ins


def _check(schema, datas, grid, fns=ALL_FNS, preds=(), oracle_preds=None, inputs=((0, False),), modes=(HG_AGG_RUNS,), maps=(), model=None):
    """every fn's per-series table == the model's, and for each (keys, groups) in maps the by-map table, for the given (flags, resident)
    inputs and modes; returns {fn: the model's per-series table}.  model: the (schema, datas) the model reads instead (the C oracle has no
    Binary columns)"""
    start, end, step, rng_ = grid
    op = oracle_preds if oracle_preds is not None else preds
    npk = getattr(schema, "npk", 2)
    handle = _handle(schema)
    ms, md = model or (schema, datas)
    exps = {}
    for fn in fns:
        exps[fn] = range_function(md, ms.arrow_schema, npk, fn, op, start, end, step, rng_)
    mexp = {(fn, j): range_function_by_map(md, ms.arrow_schema, npk, fn, keys, groups, op, start, end, step, rng_)
            for fn in fns for j, (keys, groups) in enumerate(maps)}
    for flags, resident in inputs:
        eng, ins = _engine(schema, datas, flags, resident)
        for mode in modes:
            for fn in fns:
                got = eng.scan_range_function(handle, ins, fn, preds, start, end, step, rng_, mode=mode)
                st = eng.stats()
                _same(got, exps[fn], (schema.arrow_schema.field(0).name, "t"))
                assert st["path"] == 0 and st["groups_out"] == got.num_rows, NAMES[fn]
                assert st["bytes_d2h"] == got.num_rows * (schema.arrow_schema.field(0).type.bit_width // 8 + 16)
                for j, (keys, groups) in enumerate(maps):
                    got = eng.scan_range_function_by_map(handle, ins, fn, keys, groups, preds, start, end, step, rng_, mode=mode)
                    st = eng.stats()
                    _same(got, mexp[(fn, j)], ("group", "t", "count"))
                    assert st["path"] == 0 and st["groups_out"] == got.num_rows and st["bytes_d2h"] == got.num_rows * 44
        eng.close()
    return exps


def _spread_map(n_series, G, key_lo=0):
    keys = np.arange(key_lo, key_lo + n_series, dtype=np.uint64)
    return keys, (np.arange(n_series) % G).astype(np.uint32)


# ------------------------------------------------------------------------------------------------------------------------- grids
@pytest.mark.parametrize("step,rng_", [(5_000, 2_000),        # range < step
                                       (5_000, 5_000),        # range == step
                                       (3_000, 7_777),        # range > step, not a multiple of it
                                       (0, 10_000)],          # an instant query
                         ids=str)
def test_range_function_grids(step, rng_):
    rng = np.random.default_rng(step + rng_ + 1)
    schema = _schema()
    cols = _cols(rng, 6, 50, reset_p=0.1, null_p=0.05)
    grid = (T0 + 20_000, T0 + 20_000, step, rng_) if step == 0 else (T0 - 4_000, T0 + 60_000, step, rng_)
    exps = _check(schema, [_write(schema, cols, 3)], grid, maps=[_spread_map(6, 4)], modes=(HG_AGG_RUNS, HG_AGG_HASH))
    assert exps[RATE].num_rows > 0 and exps[COUNT_OVER_TIME].num_rows > 0


def test_range_function_negative_times_and_start():
    rng = np.random.default_rng(5)
    schema = _schema(key_t=pa.int64())
    cols = _cols(rng, 5, 40, t0=-130_000, step=3000, reset_p=0.1, key_lo=-2)
    exps = _check(schema, [_write(schema, cols, 5)], (-100_001, 20_000, 7_000, 20_000))
    assert exps[RATE].num_rows > 0


@pytest.mark.parametrize("ts_t,t0,step,grid", [(pa.int32(), -30_000, 700, (-25_000, 20_000, 2_000, 5_000)),
                                                (pa.uint32(), (1 << 32) - 40_000, 500, ((1 << 32) - 30_000, (1 << 32) + 5, 2_000, 6_000)),
                                                (pa.int8(), -110, 3, (-128, 127, 5, 12))],   # 16-bit primary keys are refused by every call
                         ids=str)
def test_range_function_time_column_types(ts_t, t0, step, grid):
    rng = np.random.default_rng(step)
    schema = _schema(ts_t=ts_t)
    cols = _cols(rng, 4, 40, t0=t0, step=step, null_p=0.05)
    exps = _check(schema, [_write(schema, cols, 11)], grid)
    assert exps[RATE].num_rows > 0


def test_range_function_equal_times_under_three_primary_keys():
    """several samples at one time: a window whose samples all share one time has no rate / increase / delta / irate / idelta value"""
    rng = np.random.default_rng(7)
    schema = _schema(key_t=pa.uint32(), pk3=True)
    n = 120
    cols = {"series_id": [i // 40 for i in range(n)], "ts": [T0 + 1000 * ((i % 40) // 4) for i in range(n)], "part": [i % 4 for i in range(n)],
            "value": [float(rng.integers(0, 100)) for _ in range(n)], "tag": [0] * n}
    exps = _check(schema, [_write(schema, cols, 7)], (T0, T0 + 12_000, 1_000, 1_000))
    counts = exps[COUNT_OVER_TIME]
    assert counts.num_rows > 0 and min(counts["value"].to_pylist()) == 4.0      # every window holds the four rows of one time
    for fn in (RATE, INCREASE, DELTA, IRATE, IDELTA):
        assert exps[fn].num_rows == 0, NAMES[fn]


# ---------------------------------------------------------------------------------------------------------- extrapolation branches
def test_range_function_extrapolation_branches():
    """four samples 1 s apart (avg = 1.0, thr = 1.1 exactly the f64 of 1100 ms / 1000): at t - T0 = u, dStart = 6000 - u and dEnd = u - 3000
    ms, so u in [4000, 5000] puts both just below, on and above the threshold; the series cover the zero-point clamp (V_0 = 0, V_0 < 0,
    V_0 > 0 with a small and a large dZero, result 0 and < 0) and a reset in the first and the last pair"""
    schema = _schema()
    series = {1: [5.0, 6.0, 7.0, 8.0], 2: [0.0, 1.0, 2.0, 3.0], 3: [-2.0, 1.0, 2.0, 3.0], 4: [4.0, 4.0, 4.0, 4.0], 5: [1.0, 100.0, 101.0, 102.0],
              6: [10.0, 1.0, 2.0, 3.0], 7: [1.0, 2.0, 3.0, 0.5], 8: [9.0, 7.0, 5.0, 3.0]}
    cols = {"series_id": [], "ts": [], "value": [], "tag": []}
    for sid, vals in series.items():
        for i, v in enumerate(vals):
            cols["series_id"].append(sid)
            cols["ts"].append(T0 + 1000 * i)
            cols["value"].append(v)
            cols["tag"].append(0)
    datas = [_write(schema, cols, 40)]
    grid = (T0 + 4_000, T0 + 5_000, 1, 6_000)
    _check(schema, datas, grid, fns=(RATE, INCREASE, DELTA), maps=[(np.arange(1, 9, dtype=np.uint64), np.zeros(8, np.uint32))])
    # the grid puts dStart and dEnd one millisecond below, on and above thr, and the model takes the clamp and leaves it
    assert float(1100) / 1000 == 1.0 * 1.1 and float(1099) / 1000 < 1.1 < float(1101) / 1000
    clamp = set()
    for key, t, ts, vals in _windows(datas, schema.arrow_schema, 2, (), *grid, 2):
        _, _, d_start, _, d_zero = extrapolation(t, 6_000, [(T, float(V)) for T, V in zip(ts, vals)], True)
        if d_zero is not None:
            clamp.add(d_start == d_zero)
    assert clamp == {True, False}
    # windows of m = 1, 2, 3 samples
    _check(schema, datas, (T0, T0 + 4_000, 500, 2_500), fns=(RATE, INCREASE, DELTA, IRATE, IDELTA, RESETS, CHANGES))


@pytest.mark.parametrize("rng_", [1_001, 299_999], ids=str)
def test_range_function_range_not_whole_seconds(rng_):
    """seconds(R) of Go's Duration.Seconds for a range that is not a whole number of seconds"""
    rng = np.random.default_rng(rng_)
    schema = _schema()
    cols = _cols(rng, 3, 80, step=max(250, rng_ // 20), reset_p=0.05)
    start = T0 + rng_
    _check(schema, [_write(schema, cols, 41)], (start, start + 40 * max(250, rng_ // 20), max(250, rng_ // 20) * 3, rng_), fns=(RATE,))


def _fma_differs(t, range_ms, s):
    """would an FMA of sampled * (V_0 / result) + sampled round differently from the two rounded steps, in this window?"""
    result, sampled, d_start, d_end, d_zero = extrapolation(t, range_ms, s, True)
    if d_zero is None or d_zero != d_start:
        return False
    q = s[0][1] / result
    fused = float(Fraction(sampled) * Fraction(q) + Fraction(sampled))
    return fused != sampled + d_zero


def test_range_function_no_fused_multiply_add():
    """windows where a contracted FMA would change rate's result: short windows after frequent counter restarts (a small V_0 beside the
    increase, so the zero-point clamp takes dStart = sampled * (V_0 / result)) at jittered times"""
    rng = np.random.default_rng(43)
    schema = _schema()
    cols = _cols(rng, 8, 60, reset_p=0.5)
    datas = [_write(schema, cols, 43)]
    grid = (T0 + 1_000, T0 + 60_000, 500, 2_500)
    n_fma = sum(1 for key, t, ts, vals in _windows(datas, schema.arrow_schema, 2, (), *grid, 2)
                if len([v for v in vals if v is not None]) >= 2 and _fma_differs(t, grid[3], [(T, float(V)) for T, V in zip(ts, vals) if V is not None]))
    assert n_fma > 0
    _check(schema, datas, grid, fns=(RATE, INCREASE), maps=[_spread_map(8, 3)])


# -------------------------------------------------------------------------------------------------------------------------- values
@pytest.mark.parametrize("value_t", [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32(), pa.int64(), pa.uint64()], ids=str)
def test_range_function_integer_values_at_their_limits(value_t):
    rng = np.random.default_rng(value_t.bit_width + pa.types.is_signed_integer(value_t) + 50)
    schema = _schema(value_t=value_t)
    cols = _cols(rng, 4, 30, null_p=0.1)
    lo, hi = (-(1 << (value_t.bit_width - 1)), (1 << (value_t.bit_width - 1)) - 1) if pa.types.is_signed_integer(value_t) else (0, (1 << value_t.bit_width) - 1)
    edge = [lo, hi, lo + 1, hi - 1, 0]
    if value_t.bit_width == 64:
        edge += [(1 << 53) - 1, 1 << 53, (1 << 53) + 1]
    cols["value"] = [None if v is None else (edge[i % len(edge)] if i % 3 == 0 else lo + (int(rng.integers(0, 1 << 62)) * (hi - lo) >> 62))
                     for i, v in enumerate(cols["value"])]
    _check(schema, [_write(schema, cols, 8)], (T0, T0 + 35_000, 2_000, 9_000), maps=[_spread_map(4, 2)])


def test_range_function_float_specials_and_nulls():
    """±0.0 (changes 0), ±inf, NaN (never a reset; no change between two NaNs), NULL values in the middle and all-NULL windows (absent)"""
    schema = _schema()
    inf, nan = float("inf"), float("nan")
    rows = [(1, [None, None, None, None, None]),
            (2, [0.0, -0.0, 0.0, -0.0, 0.0]),
            (3, [1.0, nan, nan, 2.0, 0.5, -nan]),
            (4, [inf, 1.0, -inf, inf, 2.0, inf]),
            (5, [None, 3.0, None, None, 1.0, None]),
            (6, [nan, 1.0, nan, nan, 1.0, 1.0])]
    cols = {"series_id": [], "ts": [], "value": [], "tag": []}
    for sid, vals in rows:
        for i, v in enumerate(vals):
            cols["series_id"].append(sid)
            cols["ts"].append(T0 + 1000 * i)
            cols["value"].append(v)
            cols["tag"].append(0)
    datas = [_write(schema, cols, 9)]
    grid = (T0, T0 + 7_000, 1_000, 3_000)
    exps = _check(schema, datas, grid, maps=[(np.arange(1, 7, dtype=np.uint64), np.array([0, 0, 1, 1, 2, 2], np.uint32))])
    by = {(r["series_id"], r["t"]): r["value"] for r in exps[CHANGES].to_pylist()}
    assert all(v == 0.0 for (sid, _), v in by.items() if sid == 2) and not any(sid == 1 for sid, _ in by)
    assert by[(3, T0 + 2000)] == 1.0                                          # [1, nan, nan]: 1 -> nan changes, nan -> nan does not
    assert all(r["value"] == 0.0 for r in exps[RESETS].to_pylist() if r["series_id"] == 6)


def test_range_function_over_time_equals_range_aggregate():
    """*_over_time and resets are the range aggregate's columns, bit for bit (count: the non-NULL samples)"""
    rng = np.random.default_rng(45)
    schema = _schema()
    cols = _cols(rng, 5, 50, null_p=0.1, reset_p=0.1)
    datas = [_write(schema, cols, 45)]
    grid = (T0, T0 + 50_000, 2_500, 7_000)
    eng, ins = _engine(schema, datas)
    h = _handle(schema)
    agg = eng.scan_range_aggregate(h, ins, [], *grid)
    valid = agg["first_value"].is_valid().to_pylist()
    keep = [i for i, ok in enumerate(valid) if ok]
    for fn, col in ((SUM_OVER_TIME, "sum"), (MIN_OVER_TIME, "min"), (MAX_OVER_TIME, "max"), (LAST_OVER_TIME, "last_value"), (RESETS, "resets")):
        got = eng.scan_range_function(h, ins, fn, [], *grid)
        assert got["t"].to_pylist() == [agg["t"][i].as_py() for i in keep]
        want = pa.array([float(agg[col][i].as_py()) for i in keep], pa.float64())
        assert _f64_bits(got["value"].combine_chunks()) == _f64_bits(want), col
    got = eng.scan_range_function(h, ins, COUNT_OVER_TIME, [], *grid)
    full = eng.scan_range_function(h, ins, SUM_OVER_TIME, [], *grid)
    assert got.num_rows == full.num_rows and all(c >= 1.0 for c in got["value"].to_pylist())
    eng.close()


# ------------------------------------------------------------------------------------------------------------------------- by map
def test_range_function_by_map_groups():
    """several series per group in an unsorted map with same-group duplicates; series outside the map; ordinals 0 and 2^32 - 1; a group
    with no value at some t; NaN and ±inf among the summed values (their series order decides the sum)"""
    rng = np.random.default_rng(47)
    schema = _schema()
    cols = _cols(rng, 12, 40, key_lo=100, null_p=0.05, reset_p=0.1)
    for i, sid in enumerate(cols["series_id"]):
        if sid == 103 and i % 40 == 7:
            cols["value"][i] = float("nan")
        if sid == 104 and i % 40 == 11:
            cols["value"][i] = float("inf")
        if sid == 105 and i % 40 == 13:
            cols["value"][i] = -float("inf")
        if sid == 111 and 10 <= i % 40 < 30:
            cols["value"][i] = None                                           # group U32_MAX has no value in the middle
    datas = [_write(schema, cols, 47, WriteConfig(max_row_group_size=100))]
    keys = np.array([109, 100, 103, 104, 105, 101, 110, 100, 103, 111, 5, 7], np.uint64)
    groups = np.array([3, 0, 0, 0, 3, 3, 3, 0, 0, U32_MAX, 1, 1], np.uint32)   # 102, 106-108 are not in the map; 5, 7 are in no file
    grid = (T0, T0 + 40_000, 2_000, 4_000)
    for mode in (HG_AGG_RUNS, HG_AGG_HASH):
        _check(schema, datas, grid, fns=(RATE, IRATE, CHANGES, SUM_OVER_TIME, MAX_OVER_TIME), maps=[(keys, groups)], modes=(mode,),
               inputs=((0, False), (0, True)))
    exp = range_function_by_map(datas, schema.arrow_schema, 2, SUM_OVER_TIME, keys, groups, (), *grid)
    gs = exp["group"].to_pylist()
    assert set(gs) == {0, 3, U32_MAX}
    ts_max = [t for g, t in zip(gs, exp["t"].to_pylist()) if g == U32_MAX]
    assert 0 < len(ts_max) < gs.count(0)


def test_range_function_by_map_empty_map_and_pruning():
    rng = np.random.default_rng(49)
    schema = _schema()
    cols = _cols(rng, 20, 30, key_lo=0)
    datas = [_write(schema, cols, 49, WriteConfig(max_row_group_size=60))]
    grid = (T0, T0 + 30_000, 3_000, 6_000)
    eng, ins = _engine(schema, datas)
    h = _handle(schema)
    got = eng.scan_range_function_by_map(h, ins, RATE, np.zeros(0, np.uint64), np.zeros(0, np.uint32), [], *grid)
    assert got.num_rows == 0 and got.column_names == ["group", "t", "count", "sum", "min", "max"]
    got = eng.scan_range_function_by_map(h, ins, RATE, np.array([3, 4], np.uint64), np.array([1, 1], np.uint32), [], *grid)
    st = eng.stats()
    assert st["rows_decoded"] < len(cols["ts"])                                # row groups without series 3 and 4 are pruned
    exp = range_function_by_map(datas, schema.arrow_schema, 2, RATE, [3, 4], [1, 1], (), *grid)
    _same(got, exp, ("group", "t", "count"))
    assert exp.num_rows > 0 and set(exp["count"].to_pylist()) <= {1, 2}
    eng.close()


@device_only
def test_range_function_by_map_many_series():
    """4 000 series in 100 groups over 120 steps: the sum over 40 series of a group in series order, bit for bit"""
    rng = np.random.default_rng(51)
    schema = _schema()
    cols = _cols(rng, 4000, 30, step=10_000, reset_p=0.02)
    datas = [_write(schema, cols, 51, WriteConfig(max_row_group_size=8192))]
    keys, groups = _spread_map(4000, 100)
    _check(schema, datas, (T0, T0 + 300_000, 2_500, 60_000), fns=(RATE, INCREASE), maps=[(keys, groups)])


# ------------------------------------------------------------------------------------------------------------------------- inputs
def test_range_function_overwritten_rows_across_overlapping_ssts():
    rng = np.random.default_rng(13)
    schema = _schema()
    old = _cols(rng, 5, 40, jitter=False, reset_p=0.1)
    new = {k: v[::3] for k, v in old.items()}
    new["value"] = [v + 1000.0 if v is not None else None for v in new["value"]]
    datas = [_write(schema, old, 20), _write(schema, new, 21)]
    _check(schema, datas, (T0, T0 + 45_000, 4_000, 10_000), fns=(RATE, IDELTA, CHANGES, SUM_OVER_TIME), maps=[_spread_map(5, 2)],
           inputs=((0, False), (0, True), (HG_FLAG_NO_PRUNING, False)))


@pytest.mark.parametrize("codec", [ParquetCompression.Uncompressed, ParquetCompression.Snappy, ParquetCompression.Zstd])
@pytest.mark.parametrize("kind", ["plain", "delta_dict"])
def test_range_function_codecs_and_encodings(codec, kind):
    rng = np.random.default_rng(17)
    schema = _schema(value_t=pa.int64())
    cols = _cols(rng, 5, 50, ints=True, null_p=0.03)
    cols["value"] = [None if v is None else int(v) for v in cols["value"]]
    opts = {} if kind == "plain" else {"ts": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                       "series_id": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                       "value": ColumnOptions(enable_dict=True)}
    cfg = WriteConfig(compression=codec, max_row_group_size=100, column_options=opts)
    _check(schema, [_write(schema, cols, 22, cfg)], (T0 + 5_000, T0 + 50_000, 5_000, 15_000), fns=(RATE, IRATE, RESETS, MIN_OVER_TIME),
           maps=[_spread_map(5, 2)], inputs=((0, False), (0, True)))


def test_range_function_caller_predicates():
    """`tag = k`, `series_id IN_SET` and a Binary column's `=` beside the map's set and the time bounds"""
    rng = np.random.default_rng(19)
    schema = _schema()
    cols = _cols(rng, 20, 30, key_lo=1000, null_p=0.02)
    datas = [_write(schema, cols, 23, WriteConfig(max_row_group_size=200))]
    grid = (T0 + 3_000, T0 + 28_000, 2_500, 6_000)
    ids = np.unique(np.concatenate([np.arange(1000, 1020, 2), rng.integers(2_000, 10_000_000, 50_000)])).astype(np.uint64)
    maps = [_spread_map(20, 3, key_lo=1000)]
    _check(schema, datas, grid, fns=(RATE, SUM_OVER_TIME), preds=[("tag", "eq", 2)], maps=maps)
    # label = host-(series mod 3): `label = host-1` keeps the series the model keeps with `series_id IN (..)` on the same rows without labels
    lschema = _schema(extra=[pa.field("label", pa.binary())])
    lcols = dict(cols, label=[b"host-%d" % (s % 3) for s in cols["series_id"]])
    ldatas = [_write(lschema, lcols, 24, WriteConfig(max_row_group_size=200))]
    picked = [s for s in range(1000, 1020, 2) if s % 3 == 1]
    _check(lschema, ldatas, grid, fns=(RATE, SUM_OVER_TIME), preds=[("series_id", "in_set", ids), ("label", "eq", b"host-1")],
           oracle_preds=[("series_id", "in", picked)], maps=maps, model=(schema, [_write(schema, cols, 24, WriteConfig(max_row_group_size=200))]))


# ------------------------------------------------------------------------------------------------------- refusals, empty results
def _raw(eng, handle, ins, spec, rs, fn, preds=(), m=None):
    arr, keep = eng._descs(ins)
    p = _make_preds(handle.arrow_schema, preds)
    stream = ArrowArrayStream()
    rsp = C.byref(rs) if rs is not None else None
    if m is None:
        return eng._L.hg_scan_range_function(eng._h, C.byref(handle.desc), arr, C.c_size_t(len(ins)), p, C.c_size_t(len(preds)), C.byref(spec),
                                             rsp, C.c_uint32(fn), C.byref(stream))
    mp = C.byref(m) if m != "null" else None
    return eng._L.hg_scan_range_function_by_map(eng._h, C.byref(handle.desc), arr, C.c_size_t(len(ins)), p, C.c_size_t(len(preds)),
                                                C.byref(spec), rsp, C.c_uint32(fn), mp, C.byref(stream))


def test_range_function_refusals_before_device_work():
    rng = np.random.default_rng(33)
    schema = _schema(extra=[pa.field("blob", pa.binary()), pa.field("fval", pa.float32())])
    cols = _cols(rng, 3, 10)
    cols["blob"] = [b"x"] * len(cols["ts"])
    cols["fval"] = [1.0] * len(cols["ts"])
    handle = _handle(schema)
    ins = _inputs([_write(schema, cols, 33)])
    good = (T0, T0 + 10_000, 1_000, 5_000)
    m = _group_map(schema.arrow_schema, 0, [0, 1, 2], [0, 0, 1])
    dup = _group_map(schema.arrow_schema, 0, [1, 0, 1], [0, 0, 1])
    append = StorageSchema.try_new(pa.schema([pa.field("series_id", pa.uint64()), pa.field("ts", pa.int64()), pa.field("blob", pa.binary())]), 2,
                                   UpdateMode.Append)
    handle_a = SchemaHandle(append.arrow_schema, 2, UpdateMode.Append)
    eng = Engine(device=0)
    eng.scan_range_function(handle, ins, RATE, [], *good)
    before = eng.stats()
    assert before["kernel_launches"] > 0
    cases = [  # (handle, inputs, spec kwargs, range spec, fn, preds, map, code, message)
        (handle, ins, {}, good, HG_FN_LAST_OVER_TIME + 1, (), None, 1, "range function: fn is not an hg_range_fn"),               # fn outside the enum
        (handle, ins, {}, good, 1 << 31, (), m, 1, "range function: fn is not an hg_range_fn"),
        (handle, ins, {}, good, RATE, [("tag", "ge", 0)] * 7, None, 2, "more than 6 predicates (the range's time bounds take two of 8)"),  # 7 caller predicates (6 with the time bounds are accepted)
        (handle, ins, {}, good, RATE, [("tag", "ge", 0)] * 6, m, 2, "more than 5 predicates (the map's set and the range's time bounds take three of 8)"),  # 6 with a map (5 are accepted)
        (handle, ins, {}, None, RATE, (), None, 1, "null range spec"),                                                            # the range refusals
        (handle, ins, {}, (T0, T0 + 10, 0, 5), RATE, (), m, 1, "range spec: step_ms must be > 0"),
        (handle, ins, {}, (T0, T0 + 10, 1, 0), RATE, (), None, 1, "range spec: range_ms must be > 0"),
        (handle, ins, {}, (T0 + 10, T0, 1, 5), RATE, (), m, 1, "range spec: start_ms > end_ms"),
        (handle, ins, {"window_ms": 1000}, good, RATE, (), None, 1, "a range aggregate takes its windows from the range spec: window_ms must be <= 0"),
        (handle, ins, {"value_col": 4}, good, RATE, (), m, 1, "Binary columns cannot be grouped or aggregated"),                  # Binary value column
        (handle, ins, {"group_col": 3}, good, RATE, (), m, 2, "counter aggregate: the group column must be the first primary key (one series per group)"),  # not one series per window
        (handle, ins, {"ts_col": 3}, good, RATE, (), None, 2, "counter aggregate: the time column must be the second primary key (samples in time order)"),
        (handle, ins, {"mode": 2}, good, RATE, (), m, 1, "aggregation mode"),
        (handle, ins, {}, good, RATE, (), "null", 1, "null group map"),                                                           # the map refusals
        (handle, ins, {}, good, RATE, (), dup, 1, "group map: a key mapped to two different groups"),                             # a key mapped to two groups
        (handle, ins, {"group_col": 5}, good, RATE, (), m, 2, "counter aggregate: the group column must be the first primary key (one series per group)"),  # a float key column is not the series
        (handle_a, [], {"value_col": 1}, good, RATE, (), None, 2, "aggregation over an Append-mode (BytesMergeOperator) table"),  # an Append-mode table, without any SST too
        (handle_a, [], {"value_col": 1}, good, RATE, (), m, 2, "aggregation over an Append-mode (BytesMergeOperator) table"),
        (handle, ins, {}, None, HG_FN_LAST_OVER_TIME + 1, (), m, 1, "range function: fn is not an hg_range_fn"),                  # two faults: the function is reported before the range
        (handle, ins, {}, None, RATE, (), "null", 1, "null group map"),                                                           # and the null map before the range
    ]
    for h, ii, kw, grid, fn, preds, mm, code, message in cases:
        spec = HgAggSpec(kw.get("group_col", 0), kw.get("ts_col", 1), kw.get("window_ms", 0), kw.get("value_col", 2), kw.get("mode", 0))
        rc = _raw(eng, h, ii, spec, HgRangeSpec(*grid) if grid is not None else None, fn, preds, mm)
        assert rc == code, (kw, grid, fn, len(preds), rc, eng._L.hg_last_error())
        assert eng._L.hg_last_error().decode() == message, (rc, eng._L.hg_last_error())
        assert eng.stats() == before, (kw, grid, fn)
    assert eng.scan_range_function(handle, ins, RATE, [("tag", "ge", 0)] * 6, *good).num_rows > 0
    assert eng.scan_range_function_by_map(handle, ins, RATE, [0, 1, 2], [0, 0, 1], [("tag", "ge", 0)] * 5, *good).num_rows > 0
    eng.close()


def test_range_function_empty_input_and_no_passing_row():
    schema = _schema()
    rng = np.random.default_rng(35)
    data = _write(schema, _cols(rng, 3, 10), 35)
    h = _handle(schema)
    for datas, preds in (([], []), ([data], [("tag", "gt", 10)])):
        eng, ins = _engine(schema, datas)
        got = eng.scan_range_function(h, ins, RATE, preds, T0, T0 + 60_000, 1_000, 5_000)
        assert got.num_rows == 0 and got.column_names == ["series_id", "t", "value"]
        st = eng.stats()
        assert st["groups_out"] == 0 and st["bytes_d2h"] == 0
        got = eng.scan_range_function_by_map(h, ins, SUM_OVER_TIME, [0, 1, 2], [0, 1, 1], preds, T0, T0 + 60_000, 1_000, 5_000)
        assert got.num_rows == 0 and got.column_names == ["group", "t", "count", "sum", "min", "max"]
        st = eng.stats()
        assert st["groups_out"] == 0 and st["bytes_d2h"] == 0
        eng.close()
