"""Counter aggregates (`hg_scan_counter_aggregate`, `Engine.scan_counter_aggregate`): per (series, bucket) the first and last sample with a
non-NULL value, the increase with counter resets taken into account and the number of resets, computed by reduce_counter_groups_kernel on
the general pipeline's deduplicated stream.

Every case is compared with tests/counter_model.py (a sequential Python loop over the C oracle's deduplicated stream) bit for bit: keys,
buckets, counts and resets as integers, the f64 columns as bit patterns, validity included.  NaN is the one exception: IEEE leaves the
payload of a NaN result to the hardware, so a NaN matches any NaN."""
import numpy as np
import pyarrow as pa
import pytest

from counter_model import counter_aggregate
from horaedb_b200 import sstgen
from horaedb_b200._ffi import HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_FUSED, HG_FLAG_NO_PRUNING, Engine, HgError, SchemaHandle, SstInput
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode

pytestmark = pytest.mark.gpu
_ids = iter(range(150_000_000, 160_000_000))
T0 = sstgen.T0_MS
F64_COLS = ("first_value", "last_value", "increase")


def _schema(key_t=pa.uint64(), value_t=pa.float64(), ts_t=pa.int64(), mode=UpdateMode.Overwrite, extra=()):
    user = pa.schema([pa.field("series_id", key_t), pa.field("ts", ts_t), pa.field("value", value_t), pa.field("tag", pa.uint32()), *extra])
    s = StorageSchema.try_new(user, 2, mode)
    s.user = user
    return s


def _write(schema, cols, seq, cfg=None):
    batch = pa.RecordBatch.from_arrays([pa.array(cols[f.name], f.type) for f in schema.user], schema=schema.user)
    return sstgen.write_sst(schema, batch, seq=seq, cfg=cfg or WriteConfig(max_row_group_size=500))


def _counter_cols(rng, n_series, points, key_lo=0, t0=T0, step=1000, reset_p=0.05, null_p=0.0, ints=False):
    """monotone counters with random restarts (a drop to a small value) and optional NULL values"""
    sid, ts, val, tag = [], [], [], []
    for s in range(n_series):
        v = float(rng.integers(0, 100))
        for p in range(points):
            if rng.random() < reset_p:
                v = float(rng.integers(0, 5))
            else:
                v += float(rng.integers(0, 50)) if ints else float(rng.random() * 50)
            sid.append(key_lo + s)
            ts.append(t0 + p * step)
            val.append(None if rng.random() < null_p else v)
            tag.append(int(rng.integers(0, 4)))
    return {"series_id": sid, "ts": ts, "value": val, "tag": tag}


def _inputs(datas):
    return [SstInput(id=next(_ids), data=d) for d in datas]


def _run(schema, datas, preds=(), flags=0, resident=False, **kw):
    handle = SchemaHandle(schema.arrow_schema, 2, schema.update_mode)
    eng = Engine(device=0, flags=flags)
    ins = _inputs(datas)
    if resident:
        for i in range(len(ins)):
            eng.load_sst(handle, ins[i])
            ins[i] = SstInput(id=ins[i].id)
    got = eng.scan_counter_aggregate(handle, ins, preds, **kw)
    st = eng.stats()
    agg = eng.scan_aggregate(handle, ins, preds, group_col=kw.get("group_col", 0), ts_col=kw.get("ts_col", 1),
                             window_ms=kw.get("window_ms", 0), value_col=kw.get("value_col", 2))
    eng.close()
    return got, st, agg


def _f64_bits(col):
    a = col.fill_null(0.0).to_numpy().astype(np.float64)
    bits = a.view(np.uint64).copy()
    bits[np.isnan(a)] = 0x7FF8000000000000
    return bits.tolist()


def _assert_same(got, exp):
    assert got.column_names == exp.column_names
    assert got.num_rows == exp.num_rows, (got.num_rows, exp.num_rows)
    for name in exp.column_names:
        g, e = got[name].combine_chunks(), exp[name].combine_chunks()
        assert g.type == e.type, (name, g.type, e.type)
        assert g.is_valid().to_pylist() == e.is_valid().to_pylist(), name
        if name in F64_COLS:
            assert _f64_bits(g) == _f64_bits(e), name
        else:
            assert g.to_pylist() == e.to_pylist(), name


def _check(schema, datas, preds=(), window_ms=0, oracle_preds=None, modes=(HG_AGG_RUNS,), **kw):
    """the counter table == the model's, resident and transient, with and without pruning; key / bucket / count == hg_scan_aggregate's"""
    exp = counter_aggregate(datas, schema.arrow_schema, 2, oracle_preds if oracle_preds is not None else preds, window_ms=window_ms)
    for flags, resident in ((0, False), (0, True), (HG_FLAG_NO_PRUNING, False)):
        for mode in modes:
            got, st, agg = _run(schema, datas, preds, flags=flags, resident=resident, window_ms=window_ms, mode=mode, **kw)
            _assert_same(got, exp)
            assert st["path"] == 0 and st["groups_out"] == got.num_rows
            key = exp.column_names[0]
            assert got[key].to_pylist() == agg[key].to_pylist()
            assert got["count"].to_pylist() == agg["count"].to_pylist()
            if window_ms > 0:
                assert got["bucket"].to_pylist() == agg["bucket"].to_pylist()
            else:
                assert "bucket" not in got.column_names
    return exp


# ---------------------------------------------------------------------------------------------------------- resets and windows
@pytest.mark.parametrize("window_ms", [0, 7_000, 60_000])
def test_counter_resets_at_several_windows(window_ms):
    rng = np.random.default_rng(window_ms + 1)
    schema = _schema(key_t=pa.int64())
    cols = _counter_cols(rng, 12, 90, key_lo=-6, t0=-150_000, step=3000, reset_p=0.1)  # times from -150 s to +117 s: bucket 0, negatives
    exp = _check(schema, [_write(schema, cols, 3)], window_ms=window_ms, modes=(HG_AGG_RUNS, HG_AGG_HASH))
    assert sum(exp["resets"].to_pylist()) > 10
    if window_ms:
        assert 0 in exp["bucket"].to_pylist() and min(exp["bucket"].to_pylist()) < 0


@pytest.mark.parametrize("ts_t,t0,step,window_ms", [(pa.int32(), -3000, 100, 700), (pa.uint32(), (1 << 32) - 6001, 100, 700),
                                                     (pa.int8(), -60, 2, 7), (pa.uint8(), 0, 4, 50),
                                                     (pa.uint64(), (1 << 63) - 3000, 100, 1000)], ids=str)
def test_counter_time_column_types(ts_t, t0, step, window_ms):
    """first_ts / last_ts are the time column widened to i64 for every primary-key time type; u64 times from 2^63 on widen to negative
    i64 values (and buckets), as bucket_of widens them"""
    rng = np.random.default_rng(t0 & 0xFFFF)
    schema = _schema(ts_t=ts_t)
    cols = _counter_cols(rng, 5, 60, t0=t0, step=step, reset_p=0.1, null_p=0.05)
    for window in (0, window_ms):
        exp = _check(schema, [_write(schema, cols, 5)], window_ms=window)
    if ts_t == pa.uint64():
        assert min(exp["last_ts"].to_pylist()) < 0 < max(exp["first_ts"].to_pylist())


def test_counter_chain_by_hand():
    """one series with known values: increase and resets written out"""
    schema = _schema()
    vals = [5.0, 7.0, 7.0, 2.0, 3.0, 10.0, 1.0]
    cols = {"series_id": [1] * 7, "ts": [T0 + i for i in range(7)], "value": vals, "tag": [0] * 7}
    got, _, _ = _run(schema, [_write(schema, cols, 1)])
    row = got.to_pylist()[0]
    assert row["count"] == 7 and row["resets"] == 2
    assert row["increase"] == ((((((0.0 + 2.0) + 0.0) + 2.0) + 1.0) + 7.0) + 1.0)
    assert (row["first_ts"], row["first_value"], row["last_ts"], row["last_value"]) == (T0, 5.0, T0 + 6, 1.0)


# ------------------------------------------------------------------------------------------------------------ value and key types
@pytest.mark.parametrize("value_t,key_t", [(pa.uint64(), pa.uint8()), (pa.int64(), pa.int8()), (pa.int32(), pa.uint32()),
                                           (pa.float32(), pa.int64()), (pa.float64(), pa.uint64()), (pa.float64(), pa.int32())], ids=str)
def test_counter_value_and_key_types(value_t, key_t):
    """every key type a primary key may have (8, 32 and 64 bits, both signednesses; 16-bit keys are refused by every call), the
    type's edge keys, and u64 / i64 / i32 / f32 / f64 values"""
    rng = np.random.default_rng(value_t.bit_width + key_t.bit_width)
    schema = _schema(key_t=key_t, value_t=value_t)
    cols = _counter_cols(rng, 10, 60, ints=True, reset_p=0.08, null_p=0.05)
    if pa.types.is_unsigned_integer(key_t):
        cols["series_id"] = [s + (1 << key_t.bit_width) - 10 for s in cols["series_id"]]     # up to the type's maximum
    else:
        cols["series_id"] = [s - (1 << (key_t.bit_width - 1)) for s in cols["series_id"]]   # from the type's minimum
    if value_t == pa.uint64():
        cols["value"][5] = float((1 << 64) - 2048)       # above 2^53: compared as rounded f64
    elif value_t == pa.int64():
        cols["value"][5] = float(-(1 << 62))
    elif value_t == pa.int32():
        cols["value"][5] = float(-(1 << 31))
    cols["value"] = [None if v is None else (v if pa.types.is_floating(value_t) else int(v)) for v in cols["value"]]
    _check(schema, [_write(schema, cols, 4)], window_ms=20_000)


# ----------------------------------------------------------------------------------------------------------- dedup, NULL, NaN
def test_counter_overwritten_sample_causes_no_reset():
    """an older file holds a bad sample (a drop) that a newer __seq__ overwrites: only the newer value takes part"""
    schema = _schema()
    old = {"series_id": [1, 1, 1, 1, 2, 2], "ts": [T0, T0 + 1, T0 + 2, T0 + 3, T0, T0 + 1], "value": [10.0, 20.0, 5.0, 30.0, 1.0, 0.5],
           "tag": [0] * 6}
    new = {"series_id": [1, 2], "ts": [T0 + 2, T0 + 1], "value": [25.0, 2.0], "tag": [1, 1]}
    datas = [_write(schema, old, 10), _write(schema, new, 11)]
    exp = _check(schema, datas)
    assert exp["resets"].to_pylist() == [0, 0] and exp["increase"].to_pylist() == [20.0, 1.0]


def test_counter_nulls_nan_and_infinities():
    schema = _schema()
    inf = float("inf")
    rows = [(1, [None, None, None]),                                    # all NULL: first / last NULL, increase 0, resets 0
            (2, [None, 3.0, None, 1.0, None]),
            (3, [1.0, float("nan"), 2.0, 0.5]),
            (4, [inf, 1.0, -inf, inf, 2.0]),
            (5, [float("nan")]),
            (6, [-inf, -inf, 0.0])]
    cols = {"series_id": [], "ts": [], "value": [], "tag": []}
    for sid, vals in rows:
        for i, v in enumerate(vals):
            cols["series_id"].append(sid)
            cols["ts"].append(T0 + 10 * i)
            cols["value"].append(v)
            cols["tag"].append(i)
    for window in (0, 20):
        exp = _check(schema, [_write(schema, cols, 12)], window_ms=window)
    got, _, _ = _run(schema, [_write(schema, cols, 12)])
    first = got.to_pylist()[0]
    assert first["count"] == 3 and first["first_value"] is None and first["last_ts"] is None
    assert first["increase"] == 0.0 and first["resets"] == 0


# ----------------------------------------------------------------------------------------------- shapes: boundaries, codecs, encodings
def test_counter_groups_span_row_groups_and_files():
    rng = np.random.default_rng(21)
    schema = _schema()
    a = _counter_cols(rng, 6, 40, t0=T0, reset_p=0.1)
    b = _counter_cols(rng, 6, 40, t0=T0 + 40_000, reset_p=0.1)
    cfg = WriteConfig(max_row_group_size=7)
    for window in (0, 30_000):
        _check(schema, [_write(schema, a, 20, cfg), _write(schema, b, 21, cfg)], window_ms=window)


@pytest.mark.parametrize("codec", [ParquetCompression.Uncompressed, ParquetCompression.Snappy, ParquetCompression.Zstd])
@pytest.mark.parametrize("kind", ["plain", "delta_dict"])
def test_counter_codecs_and_encodings(codec, kind):
    rng = np.random.default_rng(31)
    schema = _schema(value_t=pa.int64())
    cols = _counter_cols(rng, 8, 70, ints=True, reset_p=0.05, null_p=0.03)
    cols["value"] = [None if v is None else int(v) for v in cols["value"]]
    if kind == "plain":
        cfg = WriteConfig(compression=codec, max_row_group_size=150)
    else:
        cfg = WriteConfig(compression=codec, max_row_group_size=150,
                          column_options={"ts": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                          "series_id": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                          "value": ColumnOptions(enable_dict=True)})
    _check(schema, [_write(schema, cols, 30, cfg)], window_ms=15_000)


# ------------------------------------------------------------------------------------------------------------------- predicates
def test_counter_predicates():
    """a time range, `series_id IN_SET` (10^5 ids, as an index lookup would send them) and `tag = k`; with and without pruning"""
    rng = np.random.default_rng(41)
    schema = _schema()
    cols = _counter_cols(rng, 40, 50, key_lo=1000, reset_p=0.1, null_p=0.02)
    datas = [_write(schema, cols, 40, WriteConfig(max_row_group_size=200))]
    ids = np.unique(np.concatenate([rng.choice(np.arange(1000, 1040), 15, replace=False), rng.integers(2_000, 10_000_000, 100_000)]))
    ids = ids.astype(np.uint64)
    picked = sorted(int(x) for x in ids if x < 1040)
    ts_range = [("ts", "ge", T0 + 12_000), ("ts", "lt", T0 + 37_000)]
    for window in (0, 10_000):
        _check(schema, datas, ts_range, window_ms=window)
        exp = _check(schema, datas, [("series_id", "in_set", ids), *ts_range], window_ms=window,
                     oracle_preds=[("series_id", "in", picked), *ts_range])
        assert sorted(set(exp["series_id"].to_pylist())) == picked
        _check(schema, datas, [("tag", "eq", 2)], window_ms=window)


def test_counter_transient_where_the_aggregate_ships_compressed_prefixes():
    """window 0, group = pk0 and a gate predicate on a value column of Snappy files: hg_scan_aggregate would load compressed page
    prefixes; the counter call reads whole pages, and transient equals resident"""
    rng = np.random.default_rng(51)
    schema = _schema()
    cols = _counter_cols(rng, 20, 200, reset_p=0.05)
    for i in range(len(cols["tag"])):
        cols["tag"][i] = 7 if (i % 200) < 20 else 1        # the gate passes only early in every series
    datas = [_write(schema, cols, 50, WriteConfig(compression=ParquetCompression.Snappy, max_row_group_size=1000))]
    exp = _check(schema, datas, [("tag", "eq", 7)])
    assert exp.num_rows == 20


# ------------------------------------------------------------------------------------------------------------------- stitching
def test_counter_bucket_partials_stitch_into_the_whole_range():
    """integer-valued f64 counters: the window-0 increase == sum of bucket increases + the boundary terms, exactly; resets likewise"""
    rng = np.random.default_rng(61)
    schema = _schema()
    cols = _counter_cols(rng, 9, 120, ints=True, reset_p=0.06, null_p=0.05)
    datas = [_write(schema, cols, 60, WriteConfig(max_row_group_size=111))]
    whole, _, _ = _run(schema, datas)
    parts, _, _ = _run(schema, datas, window_ms=13_000)
    by_series = {}
    for r in parts.to_pylist():
        by_series.setdefault(r["series_id"], []).append(r)
    assert len(by_series) == whole.num_rows
    for w in whole.to_pylist():
        inc, resets, last = 0.0, 0, None
        for b in by_series[w["series_id"]]:
            inc += b["increase"]
            resets += b["resets"]
            if b["first_value"] is None:
                continue
            if last is not None:
                first = b["first_value"]
                inc += first if first < last else first - last
                resets += first < last
            last = b["last_value"]
        assert inc == w["increase"] and resets == w["resets"], w["series_id"]
        assert sum(b["count"] for b in by_series[w["series_id"]]) == w["count"]


# ----------------------------------------------------------------------------------------------------------- refusals, empty results
def test_counter_refusals_before_device_work():
    rng = np.random.default_rng(71)
    schema = _schema(extra=[pa.field("blob", pa.binary()), pa.field("fval", pa.float32())])
    cols = _counter_cols(rng, 3, 10)
    cols["blob"] = [b"x"] * len(cols["ts"])
    cols["fval"] = [1.0] * len(cols["ts"])
    data = _write(schema, cols, 70)
    handle = SchemaHandle(schema.arrow_schema, 2)
    one_pk = StorageSchema.try_new(schema.user, 1)
    handle1 = SchemaHandle(one_pk.arrow_schema, 1)
    append = StorageSchema.try_new(pa.schema([pa.field("series_id", pa.uint64()), pa.field("ts", pa.int64()), pa.field("blob", pa.binary())]), 2,
                                   UpdateMode.Append)                     # every value column of an Append table is Binary
    handle_a = SchemaHandle(append.arrow_schema, 2, UpdateMode.Append)
    eng = Engine(device=0)
    ins = _inputs([data])
    eng.scan_counter_aggregate(handle, ins)
    before = eng.stats()
    assert before["kernel_launches"] > 0
    FIRST_PK = "counter aggregate: the group column must be the first primary key (one series per group)"
    SECOND_PK = "counter aggregate: the time column must be the second primary key (samples in time order)"
    cases = [(handle, dict(value_col=4), 1, "Binary columns cannot be grouped or aggregated"),  # Binary value column
             (handle, dict(value_col=-1), 1, "a counter aggregate needs a value column"),
             (handle, dict(ts_col=-1), 1, "a counter aggregate needs a time column"),
             (handle, dict(ts_col=5), 1, "time column must be an integer column"),  # a float time column
             (handle, dict(mode=2), 1, "aggregation mode"),
             (handle, dict(value_col=40), 1, "aggregation column out of range"),
             (handle, dict(group_col=3), 2, FIRST_PK),  # not one series per group
             (handle, dict(group_col=-1), 2, FIRST_PK),
             (handle, dict(ts_col=0, group_col=0), 2, SECOND_PK),
             (handle, dict(ts_col=3), 2, SECOND_PK),
             (handle1, dict(), 2, "counter aggregate: the table needs a second primary key, the time column"),
             (handle_a, dict(value_col=2), 1, "Binary columns cannot be grouped or aggregated"),
             (handle_a, dict(value_col=1), 2, "aggregation over an Append-mode (BytesMergeOperator) table")]
    for h, kw, code, msg in cases:
        with pytest.raises(HgError) as ei:
            eng.scan_counter_aggregate(h, ins, **kw)
        assert ei.value.code == code and eng._L.hg_last_error().decode() == msg, (kw, str(ei.value))
        assert eng.stats() == before, kw                 # refused before the call started: the last call's statistics are untouched
    with pytest.raises(HgError) as ei:                   # without any SST too
        eng.scan_counter_aggregate(handle_a, [], value_col=1)
    assert ei.value.code == 2 and "Append" in str(ei.value)
    assert eng.stats() == before
    eng.close()


def test_counter_empty_input_and_no_passing_row():
    schema = _schema()
    rng = np.random.default_rng(81)
    data = _write(schema, _counter_cols(rng, 3, 10), 80)
    want = {0: ["series_id", "count", "first_ts", "first_value", "last_ts", "last_value", "increase", "resets"]}
    want[60_000] = want[0][:1] + ["bucket"] + want[0][1:]
    types = {"series_id": pa.uint64(), "bucket": pa.int64(), "count": pa.uint64(), "first_ts": pa.int64(), "first_value": pa.float64(),
             "last_ts": pa.int64(), "last_value": pa.float64(), "increase": pa.float64(), "resets": pa.uint64()}
    for window in (0, 60_000):
        for datas, preds in (([], []), ([data], [("ts", "lt", T0 - 1)])):
            got, st, _ = _run(schema, datas, preds, window_ms=window)
            assert got.num_rows == 0 and got.column_names == want[window]
            assert [got.schema.field(n).type for n in got.column_names] == [types[n] for n in want[window]]
            assert st["groups_out"] == 0 and st["bytes_d2h"] == 0
            _assert_same(got, counter_aggregate(datas, schema.arrow_schema, 2, preds, window_ms=window))


def test_counter_bytes_d2h():
    schema = _schema()
    rng = np.random.default_rng(91)
    data = _write(schema, _counter_cols(rng, 5, 20, null_p=0.1), 90)
    got, st, _ = _run(schema, [data], window_ms=5_000)
    g = got.num_rows
    assert st["groups_out"] == g > 0
    assert st["bytes_d2h"] == g * 8 * 9 + (g + 7) // 8          # 9 columns of 8 bytes + the validity of first_* / last_*, once
