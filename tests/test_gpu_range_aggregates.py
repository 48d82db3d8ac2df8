"""Range-vector aggregates (`hg_scan_range_aggregate`, `hg_scan_range_quantile_aggregate`, `Engine.scan_range_aggregate` /
`scan_range_quantile_aggregate`): per series and evaluation time t_j = start + j * step, the rows with t_j - range < ts <= t_j, computed by
the range_* kernels (window enumeration, reduce_range_windows_kernel, the quantile tiers over overlapping windows) on the general pipeline.

Every case is compared with tests/range_model.py (a plain Python loop over the C oracle's deduplicated stream) bit for bit: keys, times,
counts and resets as integers, the f64 columns as bit patterns, validity included.  NaN is the one exception: IEEE leaves the payload of a
NaN result to the hardware, so a NaN matches any NaN.  Cases marked `device_only` are too large for the emulated build of the library."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pytest

from range_model import range_aggregate, range_quantile_aggregate, steps
from horaedb_b200 import sstgen
from horaedb_b200._ffi import (HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_FUSED, HG_FLAG_NO_PRUNING, ArrowArrayStream, Engine, HgAggSpec, HgError,
                               HgRangeSpec, SchemaHandle, SstInput, _make_preds)
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode

pytestmark = pytest.mark.gpu
device_only = pytest.mark.skipif("HORAE_EMU_ORDER" in os.environ, reason="too large for the emulated library")
_ids = iter(range(160_000_000, 170_000_000))
T0 = sstgen.T0_MS
INT_COLS = ("t", "count", "first_ts", "last_ts", "resets")


def _schema(key_t=pa.uint64(), value_t=pa.float64(), ts_t=pa.int64(), extra=(), pk3=False):
    fields = [pa.field("series_id", key_t), pa.field("ts", ts_t)]
    if pk3:
        fields.append(pa.field("part", pa.uint32()))
    user = pa.schema([*fields, pa.field("value", value_t), pa.field("tag", pa.uint32()), *extra])
    s = StorageSchema.try_new(user, 3 if pk3 else 2, UpdateMode.Overwrite)
    s.user = user
    s.npk = 3 if pk3 else 2
    return s


def _write(schema, cols, seq, cfg=None):
    batch = pa.RecordBatch.from_arrays([pa.array(cols[f.name], f.type) for f in schema.user], schema=schema.user)
    return sstgen.write_sst(schema, batch, seq=seq, cfg=cfg or WriteConfig(max_row_group_size=300))


def _cols(rng, n_series, points, t0=T0, step=1000, jitter=True, null_p=0.0, reset_p=0.05, ints=False, key_lo=0):
    """counters with restarts, times t0 + p * step (+ a random offset below step when jitter), optional NULL values"""
    sid, ts, val, tag = [], [], [], []
    for s in range(n_series):
        v = float(rng.integers(0, 100))
        for p in range(points):
            v = float(rng.integers(0, 5)) if rng.random() < reset_p else v + (float(rng.integers(0, 50)) if ints else float(rng.random() * 50))
            sid.append(key_lo + s)
            ts.append(t0 + p * step + (int(rng.integers(0, step)) if jitter else 0))
            val.append(None if rng.random() < null_p else v)
            tag.append(int(rng.integers(0, 4)))
    return {"series_id": sid, "ts": ts, "value": val, "tag": tag}


def _inputs(datas):
    return [SstInput(id=next(_ids), data=d) for d in datas]


def _handle(schema):
    return SchemaHandle(schema.arrow_schema, getattr(schema, "npk", 2), schema.update_mode)


def _f64_bits(col):
    a = col.fill_null(0.0).to_numpy().astype(np.float64)
    bits = a.view(np.uint64).copy()
    bits[np.isnan(a)] = 0x7FF8000000000000
    return bits.tolist()


def _assert_same(got, exp):
    assert got.column_names == exp.column_names
    assert got.num_rows == exp.num_rows, (got.num_rows, exp.num_rows)
    for i, name in enumerate(exp.column_names):
        g, e = got[name].combine_chunks(), exp[name].combine_chunks()
        assert g.type == e.type, (name, g.type, e.type)
        assert g.is_valid().to_pylist() == e.is_valid().to_pylist(), name
        if i == 0 or name in INT_COLS:
            assert g.to_pylist() == e.to_pylist(), name
        else:
            assert _f64_bits(g) == _f64_bits(e), name


def _run(schema, datas, grid, preds=(), flags=0, resident=False, quantiles=None, hbm=0, **kw):
    handle = _handle(schema)
    eng = Engine(device=0, flags=flags, hbm_budget_bytes=hbm)
    ins = _inputs(datas)
    if resident:
        for i in range(len(ins)):
            eng.load_sst(handle, ins[i])
            ins[i] = SstInput(id=ins[i].id)
    start, end, step, rng_ = grid
    if quantiles is None:
        got = eng.scan_range_aggregate(handle, ins, preds, start, end, step, rng_, **kw)
    else:
        got = eng.scan_range_quantile_aggregate(handle, ins, preds, start, end, step, rng_, quantiles=quantiles, **kw)
    st = eng.stats()
    eng.close()
    return got, st


def _check(schema, datas, grid, preds=(), oracle_preds=None, quantiles=None, inputs=((0, False), (0, True)), modes=(HG_AGG_RUNS,)):
    """the call's table == the model's, for the given (flags, resident) inputs and modes; returns the model's table"""
    start, end, step, rng_ = grid
    op = oracle_preds if oracle_preds is not None else preds
    npk = getattr(schema, "npk", 2)
    if quantiles is None:
        exp = range_aggregate(datas, schema.arrow_schema, npk, op, start, end, step, rng_)
    else:
        exp = range_quantile_aggregate(datas, schema.arrow_schema, npk, op, start, end, step, rng_, quantiles=quantiles)
    for flags, resident in inputs:
        for mode in modes:
            got, st = _run(schema, datas, grid, preds, flags=flags, resident=resident, quantiles=quantiles, mode=mode)
            _assert_same(got, exp)
            assert st["path"] == 0 and st["groups_out"] == got.num_rows
    return exp


def _both(schema, datas, grid, preds=(), **kw):
    exp = _check(schema, datas, grid, preds, **kw)
    _check(schema, datas, grid, preds, quantiles=(0.0, 0.5, 0.9, 1.0), **kw)
    return exp


# ------------------------------------------------------------------------------------------------------------------------- grids
@pytest.mark.parametrize("step,rng_", [(5_000, 2_000),        # range < step: samples in no window
                                       (5_000, 5_000),        # range == step
                                       (5_000, 25_000),       # range == 5 step
                                       (3_000, 7_777),        # range not a multiple of the step
                                       (10_000, 10_000_000)],  # range wider than the data
                         ids=str)
def test_range_grids(step, rng_):
    rng = np.random.default_rng(step + rng_)
    schema = _schema()
    cols = _cols(rng, 6, 60, reset_p=0.1, null_p=0.05)
    datas = [_write(schema, cols, 3)]
    exp = _both(schema, datas, (T0 - 4_000, T0 + 70_000, step, rng_), modes=(HG_AGG_RUNS, HG_AGG_HASH))
    assert exp.num_rows > 0
    if rng_ < step:
        assert sum(exp["count"].to_pylist()) < len(cols["ts"])
    if rng_ > step:
        assert sum(exp["count"].to_pylist()) > len(cols["ts"])


def test_range_instant_query_and_empty_grids():
    rng = np.random.default_rng(3)
    schema = _schema()
    cols = _cols(rng, 4, 40, t0=T0, step=1000, reset_p=0.1)
    gap = {k: list(v) for k, v in cols.items()}
    gap["ts"] = [t + (100_000 if i % 40 >= 20 else 0) for i, t in enumerate(cols["ts"])]   # a 100 s hole in every series
    datas = [_write(schema, gap, 4)]
    exp = _both(schema, datas, (T0 + 15_000, T0 + 15_000, 0, 10_000))                      # instant query: step is not read
    assert exp.num_rows == 4 and set(exp["t"].to_pylist()) == {T0 + 15_000}
    _both(schema, datas, (T0 + 15_000, T0 + 15_000, -7, 10_000))
    for grid in ((T0 - 900_000, T0 - 1, 60_000, 60_000),           # before the data
                 (T0 + 500_000, T0 + 900_000, 60_000, 60_000),     # after it
                 (T0 + 50_000, T0 + 110_000, 10_000, 5_000)):      # inside the hole
        exp = _both(schema, datas, grid)
        assert exp.num_rows == 0


def test_range_negative_times_and_start():
    rng = np.random.default_rng(5)
    schema = _schema(key_t=pa.int64())
    cols = _cols(rng, 5, 50, t0=-130_000, step=3000, reset_p=0.1, key_lo=-2)
    _both(schema, [_write(schema, cols, 5)], (-100_001, 20_000, 7_000, 20_000))
    _both(schema, [_write(schema, cols, 5)], (-(1 << 62), 1 << 61, 1 << 60, 1 << 60))    # huge steps and ranges: no overflow


# ---------------------------------------------------------------------------------------------------------------------- boundaries
def test_range_samples_on_window_boundaries():
    """a sample exactly on t_j is in window j; one exactly on t_j - range is not"""
    schema = _schema()
    ts = [T0 + 10_000 * i for i in range(12)]
    cols = {"series_id": [1] * 12, "ts": ts, "value": [float(i) for i in range(12)], "tag": [0] * 12}
    exp = _both(schema, [_write(schema, cols, 6)], (T0, T0 + 110_000, 10_000, 30_000))
    rows = exp.to_pylist()
    assert [r["count"] for r in rows] == [1, 2] + [3] * 10
    assert rows[5]["first_ts"] == T0 + 30_000 and rows[5]["last_ts"] == T0 + 50_000 and rows[5]["t"] == T0 + 50_000


def test_range_equal_times_within_a_series():
    """a third primary key: several rows with the same time in one series, all in the same windows, in stream order"""
    rng = np.random.default_rng(7)
    schema = _schema(key_t=pa.uint32(), pk3=True)                 # 32 + 64 + 32 bits of primary key
    n = 120
    cols = {"series_id": [i // 40 for i in range(n)], "ts": [T0 + 1000 * ((i % 40) // 4) for i in range(n)], "part": [i % 4 for i in range(n)],
            "value": [float(rng.integers(0, 100)) for _ in range(n)], "tag": [0] * n}
    _both(schema, [_write(schema, cols, 7)], (T0, T0 + 12_000, 1_000, 3_000))


# -------------------------------------------------------------------------------------------------------------------------- values
@pytest.mark.parametrize("value_t", [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32(), pa.int64(), pa.uint64()], ids=str)
def test_range_integer_values_at_their_limits(value_t):
    rng = np.random.default_rng(value_t.bit_width + pa.types.is_signed_integer(value_t))
    schema = _schema(value_t=value_t)
    cols = _cols(rng, 4, 40, null_p=0.1)
    lo, hi = (-(1 << (value_t.bit_width - 1)), (1 << (value_t.bit_width - 1)) - 1) if pa.types.is_signed_integer(value_t) else (0, (1 << value_t.bit_width) - 1)
    edge = [lo, hi, lo + 1, hi - 1, 0]
    cols["value"] = [None if v is None else (edge[i % 5] if i % 3 == 0 else lo + (int(rng.integers(0, 1 << 62)) * (hi - lo) >> 62)) for i, v in enumerate(cols["value"])]
    _both(schema, [_write(schema, cols, 8)], (T0, T0 + 45_000, 2_000, 9_000))


def test_range_float_specials_and_all_null_windows():
    schema = _schema()
    inf, nan = float("inf"), float("nan")
    rows = [(1, [None, None, None, None]),                       # windows with rows but no value: count > 0, first_* / last_* NULL
            (2, [0.0, -0.0, 0.0, -0.0, 1.0]),
            (3, [1.0, nan, 2.0, 0.5, -nan]),
            (4, [inf, 1.0, -inf, inf, 2.0]),
            (5, [None, 3.0, None, None, None, None, 1.0])]
    cols = {"series_id": [], "ts": [], "value": [], "tag": []}
    for sid, vals in rows:
        for i, v in enumerate(vals):
            cols["series_id"].append(sid)
            cols["ts"].append(T0 + 1000 * i)
            cols["value"].append(v)
            cols["tag"].append(0)
    datas = [_write(schema, cols, 9)]
    exp = _both(schema, datas, (T0, T0 + 8_000, 1_000, 2_000))
    first = [r for r in exp.to_pylist() if r["series_id"] == 1]
    assert first and all(r["count"] > 0 and r["first_value"] is None and r["last_ts"] is None for r in first)


def test_range_counter_resets_inside_and_at_a_window_start():
    """a reset in the middle of a window counts; a drop between a window's first row and the previous sample does not"""
    schema = _schema()
    vals = [10.0, 20.0, 30.0, 5.0, 15.0, 25.0, 2.0, 4.0]
    cols = {"series_id": [1] * 8, "ts": [T0 + 1000 * i for i in range(8)], "value": vals, "tag": [0] * 8}
    exp = _both(schema, [_write(schema, cols, 10)], (T0, T0 + 8_000, 1_000, 3_000))
    by_t = {r["t"]: r for r in exp.to_pylist()}
    assert by_t[T0 + 4000]["resets"] == 1 and by_t[T0 + 4000]["increase"] == 5.0 + 10.0   # [30, 5, 15]: 5 is a reset
    assert by_t[T0 + 5000]["resets"] == 0                                                         # [5, 15, 25]: the drop is before it


# ------------------------------------------------------------------------------------------------------------- time column types
@pytest.mark.parametrize("ts_t,t0,step,grid", [(pa.int64(), -50_000, 1000, (-40_000, 10_000, 3_000, 8_000)),
                                                (pa.int32(), -30_000, 700, (-25_000, 20_000, 2_000, 5_000)),
                                                (pa.int8(), -110, 3, (-128, 127, 5, 12)),   # 16-bit primary keys are refused by every call
                                                (pa.uint32(), (1 << 32) - 40_000, 500, ((1 << 32) - 30_000, (1 << 32) + 5, 2_000, 6_000)),
                                                (pa.uint8(), 0, 4, (-20, 300, 7, 30))], ids=str)
def test_range_time_column_types(ts_t, t0, step, grid):
    rng = np.random.default_rng(step)
    schema = _schema(ts_t=ts_t)
    cols = _cols(rng, 4, 60, t0=t0, step=step, null_p=0.05)
    exp = _both(schema, [_write(schema, cols, 11)], grid)
    assert exp.num_rows > 0


def test_range_u8_time_grid_below_the_domain():
    """an upper bound below an unsigned column's domain: no row passes"""
    rng = np.random.default_rng(12)
    schema = _schema(ts_t=pa.uint8())
    cols = _cols(rng, 3, 40, t0=0, step=5)
    exp = _both(schema, [_write(schema, cols, 12)], (-100, -1, 10, 50))
    assert exp.num_rows == 0


# ------------------------------------------------------------------------------------------------------------------------- inputs
def test_range_overwritten_rows_across_overlapping_ssts():
    rng = np.random.default_rng(13)
    schema = _schema()
    old = _cols(rng, 5, 50, jitter=False, reset_p=0.1)
    new = {k: v[::3] for k, v in old.items()}
    new["value"] = [v + 1000.0 if v is not None else None for v in new["value"]]
    datas = [_write(schema, old, 20), _write(schema, new, 21)]
    _both(schema, datas, (T0, T0 + 55_000, 4_000, 10_000), inputs=((0, False), (0, True), (HG_FLAG_NO_PRUNING, False)))


@pytest.mark.parametrize("codec", [ParquetCompression.Uncompressed, ParquetCompression.Snappy, ParquetCompression.Zstd])
@pytest.mark.parametrize("kind", ["plain", "delta_dict"])
def test_range_codecs_and_encodings(codec, kind):
    rng = np.random.default_rng(17)
    schema = _schema(value_t=pa.int64())
    cols = _cols(rng, 6, 60, ints=True, null_p=0.03)
    cols["value"] = [None if v is None else int(v) for v in cols["value"]]
    opts = {} if kind == "plain" else {"ts": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                       "series_id": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                       "value": ColumnOptions(enable_dict=True)}
    cfg = WriteConfig(compression=codec, max_row_group_size=100, column_options=opts)
    _both(schema, [_write(schema, cols, 22, cfg)], (T0 + 5_000, T0 + 50_000, 5_000, 15_000))


def test_range_caller_predicates():
    """`tag = k`, a time range of the caller's and `series_id IN_SET` (10^5 ids) beside the appended time bounds"""
    rng = np.random.default_rng(19)
    schema = _schema()
    cols = _cols(rng, 30, 40, key_lo=1000, null_p=0.02)
    datas = [_write(schema, cols, 23, WriteConfig(max_row_group_size=200))]
    ids = np.unique(np.concatenate([rng.choice(np.arange(1000, 1030), 10, replace=False), rng.integers(2_000, 10_000_000, 100_000)]))
    picked = sorted(int(x) for x in ids if x < 1030)
    grid = (T0 + 3_000, T0 + 38_000, 2_500, 6_000)
    _both(schema, datas, grid, [("tag", "eq", 2)])
    _both(schema, datas, grid, [("ts", "ge", T0 + 10_000), ("ts", "lt", T0 + 20_000)])
    exp = _both(schema, datas, grid, [("series_id", "in_set", ids.astype(np.uint64)), ("tag", "ne", 0)],
                oracle_preds=[("series_id", "in", picked), ("tag", "ne", 0)])
    assert sorted(set(exp["series_id"].to_pylist())) == picked


# ------------------------------------------------------------------------------------------------------------ quantile tiers
@pytest.mark.parametrize("m", [1, 2, 32, 33, 4096, 4097])
def test_range_quantile_tier_bounds(m):
    """windows of exactly m samples (and their neighbours) in every tier, overlapping by half; plus windows of NULLs only (m = 0)"""
    rng = np.random.default_rng(m)
    schema = _schema()
    n = 3 * m + 5
    vals = [float(rng.integers(-1000, 1000)) if i % 7 else float(rng.random()) for i in range(n)]
    cols = {"series_id": [1] * n + [2] * 3, "ts": [T0 + i for i in range(n)] + [T0, T0 + 1, T0 + 2], "value": vals + [None] * 3, "tag": [0] * (n + 3)}
    q = (0.0, 0.25, 0.5, 0.99, 1.0, 0.333)
    exp = _check(schema, [_write(schema, cols, 24, WriteConfig(max_row_group_size=5000))], (T0 - 1 + m, T0 + n, max(1, m // 2), m), quantiles=q)
    assert m in exp["count"].to_pylist()


@device_only
def test_range_quantile_large_windows_sharing_their_keys():
    """one series of 100 k samples, range = 40 k samples, step = 500 samples: every window is in the large tier (above kQuantileChunk),
    and neighbouring windows share 98.75 % of their keys"""
    rng = np.random.default_rng(25)
    schema = _schema()
    n = 100_000
    cols = {"series_id": [7] * n, "ts": [T0 + i for i in range(n)], "value": rng.normal(size=n).tolist(), "tag": [0] * n}
    datas = [_write(schema, cols, 25, WriteConfig(max_row_group_size=8192))]
    exp = _check(schema, datas, (T0, T0 + n, 500, 40_000), quantiles=(0.5, 0.9, 0.99), inputs=((0, True),))
    assert max(exp["count"].to_pylist()) == 40_000 and exp.num_rows == 201


# --------------------------------------------------------------------------------------------------- cross-checks with bucket calls
def test_range_equals_buckets_when_range_is_the_step():
    """range == step == w, positive times, no sample on a multiple of w: window t is bucket t - w of the bucket calls"""
    rng = np.random.default_rng(27)
    schema = _schema()
    w = 7_000
    cols = _cols(rng, 8, 80, null_p=0.05, reset_p=0.1)
    cols["ts"] = [t + 1 if t % w == 0 else t for t in cols["ts"]]
    datas = [_write(schema, cols, 27)]
    handle = _handle(schema)
    ins = _inputs(datas)
    grid = (w * (min(cols["ts"]) // w), w * (max(cols["ts"]) // w + 1), w, w)
    eng = Engine(device=0, flags=HG_FLAG_NO_FUSED)
    rg = eng.scan_range_aggregate(handle, ins, [], *grid)
    rq = eng.scan_range_quantile_aggregate(handle, ins, [], *grid, quantiles=(0.1, 0.5, 0.99))
    agg = eng.scan_aggregate(handle, ins, [], group_col=0, ts_col=1, window_ms=w, value_col=2)
    ctr = eng.scan_counter_aggregate(handle, ins, [], window_ms=w)
    qnt = eng.scan_quantile_aggregate(handle, ins, [], group_col=0, ts_col=1, window_ms=w, quantiles=(0.1, 0.5, 0.99))
    eng.close()
    buckets = [t - w for t in rg["t"].to_pylist()]
    for other in (agg, ctr, qnt):
        assert other["bucket"].to_pylist() == buckets and other["series_id"].to_pylist() == rg["series_id"].to_pylist()
        assert other["count"].to_pylist() == rg["count"].to_pylist()
    for name in ("sum", "min", "max"):
        assert _f64_bits(rg[name].combine_chunks()) == _f64_bits(agg[name].combine_chunks()), name
    for name in ("first_ts", "first_value", "last_ts", "last_value", "increase", "resets"):
        g, e = rg[name].combine_chunks(), ctr[name].combine_chunks()
        assert g.is_valid().to_pylist() == e.is_valid().to_pylist(), name
        assert g.fill_null(0).to_pylist() == e.fill_null(0).to_pylist() if name in INT_COLS else _f64_bits(g) == _f64_bits(e), name
    for j in range(3):
        g, e = rq["quantile_%d" % j].combine_chunks(), qnt["quantile_%d" % j].combine_chunks()
        assert g.is_valid().to_pylist() == e.is_valid().to_pylist() and _f64_bits(g) == _f64_bits(e)


# ------------------------------------------------------------------------------------------------- output sensitivity, pruning
def test_range_output_sensitive_over_2_24_steps():
    """1 000 sparse series x 2^24 steps in a 256 MiB budget: a dense series x steps table would need 16.8 G cells"""
    rng = np.random.default_rng(29)
    schema = _schema()
    n_series, per = 1000, 3
    cols = {"series_id": [], "ts": [], "value": [], "tag": []}
    for s in range(n_series):
        for t in sorted(rng.choice(1 << 24, per, replace=False).tolist()):
            cols["series_id"].append(s)
            cols["ts"].append(int(t))
            cols["value"].append(float(rng.integers(0, 100)))
            cols["tag"].append(0)
    datas = [_write(schema, cols, 29, WriteConfig(max_row_group_size=4096))]
    grid = (0, (1 << 24) - 1, 1, 5)
    assert steps(*grid[:3]) == 1 << 24
    exp = range_aggregate(datas, schema.arrow_schema, 2, (), *grid)
    got, st = _run(schema, datas, grid, hbm=256 << 20)
    _assert_same(got, exp)
    assert got.num_rows <= n_series * per * 5


def test_range_prunes_row_groups_outside_the_grid():
    rng = np.random.default_rng(31)
    schema = _schema()
    cols = _cols(rng, 1, 3000, step=1000, jitter=False)
    datas = [_write(schema, cols, 31, WriteConfig(max_row_group_size=250))]
    grid = (T0 + 1_000_000, T0 + 1_500_000, 60_000, 120_000)
    exp = _check(schema, datas, grid)
    got, st = _run(schema, datas, grid)
    assert st["rows_in_files"] == 3000 and st["rows_decoded"] <= 1000     # 4 of 12 row groups overlap (880 s, 1500 s]
    passing = sum(1 for t in cols["ts"] if grid[0] - grid[3] < t <= grid[1])
    assert st["rows_filtered"] == passing and st["rows_out"] == passing
    assert st["groups_out"] == got.num_rows == exp.num_rows == 9 and st["path"] == 0
    w = got.num_rows
    assert st["bytes_d2h"] == w * 8 * 12 + (w + 7) // 8          # key, t and ten columns of 8 bytes + the validity of first_* / last_*, once


# ------------------------------------------------------------------------------------------------------- refusals, empty results
def _raw_call(eng, handle, ins, spec, rs, preds=(), quantiles=None):
    arr, keep = eng._descs(ins)
    p = _make_preds(handle.arrow_schema, preds)
    stream = ArrowArrayStream()
    rsp = C.byref(rs) if rs is not None else None
    if quantiles is None:
        return eng._L.hg_scan_range_aggregate(eng._h, C.byref(handle.desc), arr, C.c_size_t(len(ins)), p, C.c_size_t(len(preds)), C.byref(spec),
                                              rsp, C.byref(stream))
    qs = (C.c_double * max(1, len(quantiles)))(*quantiles)
    return eng._L.hg_scan_range_quantile_aggregate(eng._h, C.byref(handle.desc), arr, C.c_size_t(len(ins)), p, C.c_size_t(len(preds)),
                                                   C.byref(spec), rsp, qs, C.c_uint32(len(quantiles)), C.byref(stream))


def test_range_refusals_before_device_work():
    assert C.sizeof(HgRangeSpec) == 32
    rng = np.random.default_rng(33)
    schema = _schema(extra=[pa.field("blob", pa.binary()), pa.field("fval", pa.float32())])
    cols = _cols(rng, 3, 10)
    cols["blob"] = [b"x"] * len(cols["ts"])
    cols["fval"] = [1.0] * len(cols["ts"])
    handle = _handle(schema)
    ins = _inputs([_write(schema, cols, 33)])
    u64 = _schema(ts_t=pa.uint64())
    ins64 = _inputs([_write(u64, _cols(rng, 2, 5), 34)])
    append = StorageSchema.try_new(pa.schema([pa.field("series_id", pa.uint64()), pa.field("ts", pa.int64()), pa.field("blob", pa.binary())]), 2,
                                   UpdateMode.Append)
    good = (T0, T0 + 10_000, 1_000, 5_000)
    eng = Engine(device=0)
    eng.scan_range_aggregate(handle, ins, [], *good)
    before = eng.stats()
    assert before["kernel_launches"] > 0
    I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
    seven = [("tag", "ge", 0)] * 7
    cases = [  # (handle, inputs, spec kwargs, range spec, preds, quantiles, code, message)
        (handle, ins, {}, None, (), None, 1, "null range spec"),                                                    # null range
        (handle, ins, {}, (T0, T0 + 10, 0, 5), (), None, 1, "range spec: step_ms must be > 0"),                     # step 0 with start != end
        (handle, ins, {}, (T0, T0 + 10, -1, 5), (), None, 1, "range spec: step_ms must be > 0"),
        (handle, ins, {}, (T0, T0 + 10, 1, 0), (), None, 1, "range spec: range_ms must be > 0"),                    # range 0
        (handle, ins, {}, (T0, T0, 1, -5), (), None, 1, "range spec: range_ms must be > 0"),
        (handle, ins, {}, (T0 + 10, T0, 1, 5), (), None, 1, "range spec: start_ms > end_ms"),                       # start > end
        (handle, ins, {}, (0, 1 << 24, 1, 5), (), None, 1, "range spec: more than HG_MAX_RANGE_STEPS steps"),       # 2^24 + 1 steps
        (handle, ins, {}, (I64_MIN + 4, 0, 1 << 40, 5), (), None, 1, "range spec: start_ms - range_ms or (end_ms - start_ms) + range_ms does not fit in i64"),  # start - range below i64
        (handle, ins, {}, (-(1 << 62), 1 << 62, 1 << 40, 1 << 62), (), None, 1, "range spec: start_ms - range_ms or (end_ms - start_ms) + range_ms does not fit in i64"),  # (end - start) + range above i64
        (handle, ins, {}, (I64_MIN, I64_MAX, 1 << 62, 1), (), None, 1, "range spec: start_ms - range_ms or (end_ms - start_ms) + range_ms does not fit in i64"),
        (handle, ins, {"value_col": 4}, good, (), None, 1, "Binary columns cannot be grouped or aggregated"),       # Binary value column
        (handle, ins, {"value_col": -1}, good, (), None, 1, "a counter aggregate needs a value column"),
        (handle, ins, {"window_ms": 1000}, good, (), None, 1, "a range aggregate takes its windows from the range spec: window_ms must be <= 0"),
        (handle, ins, {"mode": 2}, good, (), None, 1, "aggregation mode"),
        (handle, ins, {}, good, (), (), 1, "a quantile aggregate takes 1 to 16 quantiles"),                         # the quantile checks
        (handle, ins, {}, good, (), (1.5,), 1, "a quantile must lie in [0, 1]"),
        (handle, ins, {}, good, (), (float("nan"),), 1, "a quantile must lie in [0, 1]"),
        (handle, ins, {}, good, (), (0.5,) * 17, 1, "a quantile aggregate takes 1 to 16 quantiles"),
        (handle, ins, {"group_col": 3}, good, (), None, 2, "counter aggregate: the group column must be the first primary key (one series per group)"),  # not one series per window
        (handle, ins, {"group_col": -1}, good, (), None, 2, "counter aggregate: the group column must be the first primary key (one series per group)"),
        (handle, ins, {"ts_col": 4}, good, (), None, 1, "time column must be an integer column"),                   # a Binary time column
        (handle, ins, {"ts_col": 5}, good, (), None, 1, "time column must be an integer column"),                   # a float time column
        (handle, ins, {"ts_col": 3}, good, (), None, 2, "counter aggregate: the time column must be the second primary key (samples in time order)"),  # tag is not the second primary key
        (_handle(u64), ins64, {}, good, (), None, 2, "range aggregate on a u64 time column: times from 2^63 on do not keep their order in i64"),  # u64 time column
        (SchemaHandle(append.arrow_schema, 2, UpdateMode.Append), ins, {"value_col": 1}, good, (), None, 2, "aggregation over an Append-mode (BytesMergeOperator) table"),
        (SchemaHandle(append.arrow_schema, 2, UpdateMode.Append), [], {"value_col": 1}, good, (), None, 2, "aggregation over an Append-mode (BytesMergeOperator) table"),  # without any SST too
        (SchemaHandle(append.arrow_schema, 2, UpdateMode.Append), [], {"value_col": 1}, good, (), (0.5,), 2, "aggregation over an Append-mode (BytesMergeOperator) table"),
        (handle, ins, {}, good, seven, None, 2, "more than 6 predicates (the range's time bounds take two of 8)"),  # 7 caller predicates
        (handle, ins, {}, None, (), (1.5,), 1, "a quantile must lie in [0, 1]"),                                    # two faults: the quantiles before the range
    ]
    for h, ii, kw, grid, preds, qs, code, message in cases:
        spec = HgAggSpec(kw.get("group_col", 0), kw.get("ts_col", 1), kw.get("window_ms", 0), kw.get("value_col", 2), kw.get("mode", 0))
        rc = _raw_call(eng, h, ii, spec, HgRangeSpec(*grid) if grid is not None else None, preds, qs)
        assert rc == code, (kw, grid, len(preds), qs, rc, eng._L.hg_last_error())
        assert eng._L.hg_last_error().decode() == message, (rc, eng._L.hg_last_error())
        assert eng.stats() == before, (kw, grid)         # refused before the call started: the last call's statistics are untouched
    with pytest.raises(HgError):
        eng.scan_range_aggregate(handle, ins, [], T0, T0 + 10, 0, 5)
    six = eng.scan_range_aggregate(handle, ins, [("tag", "ge", 0)] * 6, *good)  # 6 caller predicates are accepted
    assert six.num_rows > 0
    eng.close()


def test_range_empty_input_and_no_passing_row():
    schema = _schema()
    rng = np.random.default_rng(35)
    data = _write(schema, _cols(rng, 3, 10), 35)
    names = ["series_id", "t", "count", "sum", "min", "max", "first_ts", "first_value", "last_ts", "last_value", "increase", "resets"]
    for datas, preds in (([], []), ([data], [("tag", "gt", 10)])):
        for qs in (None, (0.5, 0.9)):
            got, st = _run(schema, datas, (T0, T0 + 60_000, 1_000, 5_000), preds, quantiles=qs)
            assert got.num_rows == 0
            assert got.column_names == (names if qs is None else names[:3] + ["quantile_0", "quantile_1"])
            assert st["groups_out"] == 0 and st["bytes_d2h"] == 0
