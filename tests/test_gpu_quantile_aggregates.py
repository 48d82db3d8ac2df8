"""Quantile aggregates (`hg_scan_quantile_aggregate`, `Engine.scan_quantile_aggregate`): exact, interpolated quantiles of a value column per
(group, bucket), selected on the device from the general pipeline's deduplicated groups (the quantile_* kernels of kernels.cu).

Every case is compared with tests/quantile_model.py (sorted Python lists over the C oracle's deduplicated stream): the quantile columns as
f64 bit patterns with their NULL masks, the key / bucket / count columns as values, and those three also against `scan_aggregate` under
HG_FLAG_NO_FUSED.  NaN is the one exception to bit equality: IEEE leaves the payload of a NaN result to the hardware, so a NaN matches any
NaN (which value a rank selects still depends on the NaNs' order).

The tiers of the quantile kernels by a group's count m of non-NULL values: small m <= 32, medium m <= 4096, large above, and a large group above
16384 spans several blocks per radix pass (kernels.h: kQuantileSmallMax, kQuantileMediumMax, kQuantileChunk)."""
import math
from fractions import Fraction

import numpy as np
import pyarrow as pa
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_FUSED, HG_FLAG_NO_PRUNING, Engine, HgError, SchemaHandle, SstInput
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode
from quantile_model import quantile_aggregate

pytestmark = pytest.mark.gpu
_ids = iter(range(160_000_000, 170_000_000))
T0 = sstgen.T0_MS
SMALL_MAX, MEDIUM_MAX, CHUNK = 32, 4096, 16384
Q6 = (0.0, 0.25, 0.5, 0.9, 0.99, 1.0)


def _schema(key_t=pa.uint64(), value_t=pa.float64(), ts_t=pa.int64(), mode=UpdateMode.Overwrite, extra=()):
    user = pa.schema([pa.field("series_id", key_t), pa.field("ts", ts_t), pa.field("value", value_t), pa.field("tag", pa.uint32()), *extra])
    s = StorageSchema.try_new(user, 2, mode)
    s.user = user
    return s


def _write(schema, cols, seq, cfg=None):
    batch = pa.RecordBatch.from_arrays([pa.array(cols[f.name], f.type) for f in schema.user], schema=schema.user)
    return sstgen.write_sst(schema, batch, seq=seq, cfg=cfg or WriteConfig(max_row_group_size=500))


def _gauge_cols(rng, sizes, key_lo=0, t0=T0, step=1000, null_p=0.0, ints=False, n_tags=4):
    """series s has sizes[s] samples `step` ms apart; values random (integers when `ints`), NULL with probability null_p"""
    sid, ts, val, tag = [], [], [], []
    for s, n in enumerate(sizes):
        v = rng.integers(-1000, 1000, n) if ints else rng.normal(50.0, 20.0, n)
        nulls = rng.random(n) < null_p
        sid += [key_lo + s] * n
        ts += [t0 + p * step for p in range(n)]
        val += [None if nulls[p] else (int(v[p]) if ints else float(v[p])) for p in range(n)]
        tag += rng.integers(0, n_tags, n).tolist()
    return {"series_id": sid, "ts": ts, "value": val, "tag": tag}


def _inputs(datas):
    return [SstInput(id=next(_ids), data=d) for d in datas]


def _engine(handle, datas, flags, resident):
    eng = Engine(device=0, flags=flags)
    ins = _inputs(datas)
    if resident:
        for i in range(len(ins)):
            eng.load_sst(handle, ins[i])
            ins[i] = SstInput(id=ins[i].id)
    return eng, ins


def _run(schema, datas, preds=(), flags=0, resident=False, **kw):
    """the quantile table and its statistics, and scan_aggregate's table for the same spec under HG_FLAG_NO_FUSED"""
    handle = SchemaHandle(schema.arrow_schema, 2, schema.update_mode)
    eng, ins = _engine(handle, datas, flags, resident)
    got = eng.scan_quantile_aggregate(handle, ins, preds, **kw)
    st = eng.stats()
    eng.set_flags(flags | HG_FLAG_NO_FUSED)
    agg = eng.scan_aggregate(handle, ins, preds, group_col=kw.get("group_col", 0), ts_col=kw.get("ts_col", -1),
                             window_ms=kw.get("window_ms", 0), value_col=kw.get("value_col", 2), mode=kw.get("mode", HG_AGG_RUNS))
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
        if name.startswith("quantile_"):
            assert _f64_bits(g) == _f64_bits(e), name
        else:
            assert g.to_pylist() == e.to_pylist(), name


def _check(schema, datas, preds=(), oracle_preds=None, modes=(HG_AGG_RUNS,), quantiles=Q6, transient_only=False, model_input=None, **kw):
    """the quantile table == the model's, transient and resident, with and without pruning, in every mode given; key / bucket / count ==
    scan_aggregate's under HG_FLAG_NO_FUSED.  model_input: (schema, datas, preds) the model reads instead (the C oracle has no Binary
    columns)"""
    kw.setdefault("ts_col", 1)
    runs = ((0, False),) if transient_only else ((0, False), (0, True), (HG_FLAG_NO_PRUNING, False))
    m_schema, m_datas, m_preds = model_input or (schema, datas, oracle_preds if oracle_preds is not None else preds)
    for mode in modes:
        exp = quantile_aggregate(m_datas, m_schema.arrow_schema, 2, m_preds, mode=mode, quantiles=quantiles, **kw)
        for flags, resident in runs:
            got, st, agg = _run(schema, datas, preds, flags=flags, resident=resident, mode=mode, quantiles=quantiles, **kw)
            _assert_same(got, exp)
            assert st["path"] == 0 and st["groups_out"] == got.num_rows
            for name in got.column_names:
                if not name.startswith("quantile_"):
                    assert got[name].to_pylist() == agg[name].to_pylist(), name
    return exp


# ------------------------------------------------------------------------------------------------------------------ q sets, windows
@pytest.mark.parametrize("qs", [Q6, (0.9, 0.1, 0.9, 0.5, 0.1), (0.5,), tuple(i / 15 for i in range(16))], ids=["six", "dup_unsorted", "one", "sixteen"])
@pytest.mark.parametrize("window_ms", [0, 7_000, 60_000])
def test_quantile_sets_and_windows(qs, window_ms):
    rng = np.random.default_rng(window_ms + len(qs))
    schema = _schema(key_t=pa.int64())
    cols = _gauge_cols(rng, [3, 40, 90, 1, 2, 17], key_lo=-3, t0=-45_000, null_p=0.05)   # times from -45 s: bucket 0 and negative buckets
    _check(schema, [_write(schema, cols, 3)], quantiles=qs, window_ms=window_ms, modes=(HG_AGG_RUNS, HG_AGG_HASH))


def test_quantile_ends_are_min_and_max():
    """on NaN-free data q = 0 / 1 are scan_aggregate's min / max"""
    rng = np.random.default_rng(5)
    schema = _schema()
    cols = _gauge_cols(rng, [1, 7, 33, 300, 5000])
    for window in (0, 60_000):
        got, _, agg = _run(schema, [_write(schema, cols, 4)], ts_col=1, window_ms=window, quantiles=(1.0, 0.0))
        assert got["quantile_0"].to_pylist() == agg["max"].to_pylist()
        assert got["quantile_1"].to_pylist() == agg["min"].to_pylist()


# ------------------------------------------------------------------------------------------------------------------ value domain
INT_TYPES = [pa.uint8(), pa.int8(), pa.uint16(), pa.int16(), pa.uint32(), pa.int32(), pa.uint64(), pa.int64()]


@pytest.mark.parametrize("value_t", INT_TYPES + [pa.float32(), pa.float64()], ids=str)
def test_quantile_value_types(value_t):
    """every integer type from its minimum to its maximum, f32 and f64; group sizes in the small and medium tiers"""
    rng = np.random.default_rng(value_t.bit_width)
    schema = _schema(value_t=value_t)
    sizes = [5, 31, 120]
    cols = _gauge_cols(rng, sizes, null_p=0.05)
    n = len(cols["value"])
    if pa.types.is_integer(value_t):
        info = np.iinfo(value_t.to_pandas_dtype())
        lo, hi = int(info.min), int(info.max)
        vals = [int(x) for x in rng.integers(lo, hi, n, dtype=np.int64 if lo < 0 else np.uint64, endpoint=True)]
        vals[0], vals[1], vals[6], vals[7] = lo, hi, hi, lo
    else:
        vals = [float(x) for x in rng.normal(0, 1e3, n)]
        vals[0], vals[1] = -0.0, 0.0
    cols["value"] = [None if cols["value"][i] is None else vals[i] for i in range(n)]
    _check(schema, [_write(schema, cols, 5)], window_ms=30_000)


def test_quantile_integers_around_2_to_53_and_the_64_bit_limits():
    """i64 / u64 values above 2^53 round on their way to f64 after the selection"""
    for value_t, base in ((pa.int64(), [(1 << 53) - 2, (1 << 53) + 1, (1 << 53) + 3, -(1 << 63), (1 << 63) - 1, -(1 << 53) - 1]),
                          (pa.uint64(), [(1 << 53) - 1, (1 << 53) + 1, (1 << 64) - 1, (1 << 64) - 2049, 0, (1 << 63) + 1])):
        schema = _schema(value_t=value_t)
        vals = base * 7
        cols = {"series_id": [1] * 6 + [2] * 36, "ts": [T0 + i for i in range(42)], "value": vals, "tag": [0] * 42}
        _check(schema, [_write(schema, cols, 6)], quantiles=(0.0, 0.1, 0.33, 0.5, 0.77, 1.0))


def _f64(bits):
    return float(np.array([bits], dtype=np.uint64).view(np.float64)[0])


def test_quantile_float_edges():
    """+-0.0, +-inf, NaNs of both signs with payloads and subnormals order by IEEE totalOrder: -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf
    < +NaN; a q that lands between two NaNs, or between a NaN and a number, is NaN"""
    schema = _schema()
    inf = float("inf")
    nan_pos, nan_pay, nan_neg, nan_neg_pay = _f64(0x7FF8000000000000), _f64(0x7FF0000000000123), _f64(0xFFF8000000000000), _f64(0xFFF00000000000AB)
    sub, sub_neg = _f64(1), _f64(0x800000000000000F)
    groups = [[0.0, -0.0, 0.0, -0.0], [inf, -inf, 1.0, -1.0, 0.0], [nan_pos, 1.0, 2.0, 3.0, nan_neg], [sub, sub_neg, 0.0, -0.0, _f64(2)],
              [nan_pay, nan_neg_pay, inf, -inf, 5.0, sub], [-inf, -inf, inf, inf], [nan_neg, nan_neg, nan_neg, 1.0, 2.0, 3.0, 4.0]]
    cols = {"series_id": [], "ts": [], "value": [], "tag": []}
    for s, vals in enumerate(groups):
        for i, v in enumerate(vals):
            cols["series_id"].append(s)
            cols["ts"].append(T0 + i)
            cols["value"].append(v)
            cols["tag"].append(0)
    exp = _check(schema, [_write(schema, cols, 7)], quantiles=(0.0, 0.1, 0.25, 0.5, 0.75, 0.9, 1.0))
    rows = exp.to_pylist()
    assert str(rows[0]["quantile_0"]) == "-0.0" and str(rows[0]["quantile_6"]) == "0.0"
    assert rows[1]["quantile_0"] == -inf and rows[1]["quantile_6"] == inf
    assert rows[6]["quantile_6"] == 4.0 and np.isnan(rows[6]["quantile_0"])


def test_quantile_f32_edges():
    schema = _schema(value_t=pa.float32())
    inf = float("inf")
    sub = float(np.array([1], dtype=np.uint32).view(np.float32)[0])
    vals = [-0.0, 0.0, inf, -inf, sub, -sub, 1.5, 3.25e38, -3.25e38, 1e-30]
    cols = {"series_id": [1] * 10, "ts": [T0 + i for i in range(10)], "value": vals, "tag": [0] * 10}
    _check(schema, [_write(schema, cols, 8)], quantiles=(0.0, 0.05, 0.3, 0.5, 0.61, 0.95, 1.0))


def test_quantile_interpolation_is_not_contracted():
    """groups of two values a < b, half of each, and a q whose lo / hi fall on the last a and the first b: the interpolation differs
    when either product is fused with the addition.  One group per tier (small, medium, large split across blocks)."""
    a, b = 13386.714285714286, 14262.666666666666
    schema = _schema()
    for size, q in ((2, 0.7), (40, 0.48796153846153845), (40_000, 0.49999116227905693)):
        rank = q * (size - 1)
        w = rank - math.floor(rank)
        assert math.floor(rank) == size // 2 - 1
        plain = a * (1 - w) + b * w
        fused = (float(Fraction(a) * Fraction(1 - w) + Fraction(b * w)), float(Fraction(b) * Fraction(w) + Fraction(a * (1 - w))))
        assert plain not in fused
        vals = [a] * (size // 2) + [b] * (size - size // 2)
        cols = {"series_id": [1] * size, "ts": [T0 + i for i in range(size)], "value": vals[::-1], "tag": [0] * size}
        got, _, _ = _run(schema, [_write(schema, cols, 9, WriteConfig(max_row_group_size=50_000))], quantiles=(q,))
        assert got["quantile_0"].to_pylist() == [plain], size


# ------------------------------------------------------------------------------------------------------------------------- tiers
TIER_SIZES = [1, 2, 3, 31, 32, 33, 64, 700, MEDIUM_MAX, MEDIUM_MAX + 1, 9000, CHUNK, CHUNK + 1, 2 * CHUNK + 1234]


def test_quantile_every_tier_in_one_call():
    """groups whose m is 0 (all NULL), 1 and 2, both sides of each tier bound and a group that spans three blocks a radix pass"""
    rng = np.random.default_rng(11)
    schema = _schema()
    cols = _gauge_cols(rng, [4] + TIER_SIZES, step=1)
    cols["value"][:4] = [None] * 4
    datas = [_write(schema, cols, 11, WriteConfig(max_row_group_size=5000))]
    exp = _check(schema, datas, quantiles=(0.0, 0.01, 0.5, 0.99, 1.0, 0.5), transient_only=True)
    assert exp["count"].to_pylist() == [4] + TIER_SIZES
    assert exp["quantile_0"].to_pylist()[0] is None


def test_quantile_large_groups_with_nulls_and_ties():
    """large groups of few distinct values (every radix digit ties) with NULLs in between, in RUNS and HASH, with buckets"""
    rng = np.random.default_rng(12)
    schema = _schema(value_t=pa.int32())
    cols = _gauge_cols(rng, [CHUNK + 5000, 6000, 20], step=1, null_p=0.2, ints=True)
    cols["value"] = [None if v is None else v % 3 for v in cols["value"]]
    _check(schema, [_write(schema, cols, 12, WriteConfig(max_row_group_size=4000))], window_ms=7_000, modes=(HG_AGG_RUNS, HG_AGG_HASH),
           transient_only=True)


def test_quantile_launches_only_the_tiers_it_needs():
    """a call whose groups are all small launches fewer kernels than one that also has a large group (16 more: 8 radix passes)"""
    rng = np.random.default_rng(13)
    schema = _schema()
    small = _write(schema, _gauge_cols(rng, [20] * 50, step=1), 13)
    large = _write(schema, _gauge_cols(rng, [20] * 49 + [CHUNK + 10], step=1), 14)
    _, st_small, _ = _run(schema, [small])
    _, st_large, _ = _run(schema, [large])
    assert st_small["kernel_launches"] < st_large["kernel_launches"]
    assert st_large["kernel_launches"] - st_small["kernel_launches"] >= 16


def test_quantile_global_group_of_millions():
    """group_col = -1: one group of 3 M rows, selected by many blocks per pass"""
    rng = np.random.default_rng(14)
    schema = _schema()
    n = 3_000_000
    cols = {"series_id": np.repeat(np.arange(30, dtype=np.uint64), n // 30), "ts": np.tile(T0 + np.arange(n // 30, dtype=np.int64), 30),
            "value": rng.normal(100.0, 30.0, n), "tag": rng.integers(0, 4, n, dtype=np.uint32)}
    cols["value"][::97] = np.nan
    batch = pa.RecordBatch.from_arrays([pa.array(cols[f.name], f.type) for f in schema.user], schema=schema.user)
    data = sstgen.write_sst(schema, batch, seq=15, cfg=WriteConfig(max_row_group_size=1 << 20))
    qs = (0.0, 0.5, 0.9, 0.99, 0.999, 1.0)
    got, st, agg = _run(schema, [data], group_col=-1, quantiles=qs)
    assert got.column_names == ["count"] + ["quantile_%d" % j for j in range(len(qs))]
    assert got["count"].to_pylist() == agg["count"].to_pylist() == [n]
    v = np.sort(cols["value"][~np.isnan(cols["value"])])
    vals = v.tolist() + [float("nan")] * int(np.isnan(cols["value"]).sum())     # +NaN sorts last
    from quantile_model import quantiles_of
    exp = quantiles_of(vals, pa.float64(), qs)
    assert _f64_bits(pa.chunked_array([got["quantile_%d" % j].combine_chunks() for j in range(len(qs))]).combine_chunks()) == \
        _f64_bits(pa.array(exp, pa.float64()))


# ---------------------------------------------------------------------------------------------------- grouping, dedup, predicates
def test_quantile_hash_on_tag_and_bucket_with_nulls():
    """HASH on a key that is not the sort prefix, (tag, bucket), values with NULLs; RUNS on the same spec cuts runs of the stream"""
    rng = np.random.default_rng(21)
    schema = _schema()
    cols = _gauge_cols(rng, [300] * 8, step=250, null_p=0.15, n_tags=5)
    _check(schema, [_write(schema, cols, 21, WriteConfig(max_row_group_size=333))], group_col=3, window_ms=60_000,
           modes=(HG_AGG_HASH, HG_AGG_RUNS))
    _check(schema, [_write(schema, cols, 21)], group_col=3, window_ms=0, modes=(HG_AGG_HASH,))


def test_quantile_global_group_with_windows():
    rng = np.random.default_rng(22)
    schema = _schema()
    cols = _gauge_cols(rng, [200] * 6, step=400, null_p=0.05)
    _check(schema, [_write(schema, cols, 22)], group_col=-1, window_ms=7_000, modes=(HG_AGG_HASH, HG_AGG_RUNS))
    _check(schema, [_write(schema, cols, 22)], group_col=-1, window_ms=0)


def test_quantile_overwritten_value_does_not_count():
    """an older file holds an outlier that a newer __seq__ overwrites: only the newer value takes part"""
    schema = _schema()
    old = {"series_id": [1] * 5 + [2] * 3, "ts": [T0 + i for i in range(5)] + [T0, T0 + 1, T0 + 2],
           "value": [1.0, 2.0, 1e9, 4.0, 5.0, 7.0, -1e9, 9.0], "tag": [0] * 8}
    new = {"series_id": [1, 2], "ts": [T0 + 2, T0 + 1], "value": [3.0, None], "tag": [1, 1]}
    datas = [_write(schema, old, 30), _write(schema, new, 31)]
    exp = _check(schema, datas, quantiles=(0.0, 0.5, 1.0))
    assert exp["quantile_2"].to_pylist() == [5.0, 9.0] and exp["quantile_0"].to_pylist() == [1.0, 7.0]
    assert exp["count"].to_pylist() == [5, 3]


def test_quantile_predicates():
    """a time range, `series_id IN_SET` (10^5 ids) and a Binary predicate on another column; with and without pruning"""
    rng = np.random.default_rng(41)
    schema = _schema(extra=[pa.field("label", pa.binary())])
    cols = _gauge_cols(rng, [50] * 40, key_lo=1000, null_p=0.05)
    cols["label"] = [b"host-%d" % (i % 3) for i in range(len(cols["ts"]))]
    datas = [_write(schema, cols, 40, WriteConfig(max_row_group_size=200))]
    ids = np.unique(np.concatenate([rng.choice(np.arange(1000, 1040), 15, replace=False), rng.integers(2_000, 10_000_000, 100_000)]))
    ids = ids.astype(np.uint64)
    picked = sorted(int(x) for x in ids if x < 1040)
    ts_range = [("ts", "ge", T0 + 12_000), ("ts", "lt", T0 + 37_000)]
    # the model reads the same rows without the Binary column (the C oracle has none); for the label predicate, the rows it keeps
    # (one file: no older versions to uncover)
    plain = _schema()
    names = ("series_id", "ts", "value", "tag")
    whole = [_write(plain, {k: cols[k] for k in names}, 40)]
    keep = [i for i, x in enumerate(cols["label"]) if x == b"host-1"]
    labelled = [_write(plain, {k: [cols[k][i] for i in keep] for k in names}, 40)]
    for window in (0, 10_000):
        _check(schema, datas, ts_range, window_ms=window, model_input=(plain, whole, ts_range))
        exp = _check(schema, datas, [("series_id", "in_set", ids), *ts_range], window_ms=window,
                     model_input=(plain, whole, [("series_id", "in", picked), *ts_range]))
        assert sorted(set(exp["series_id"].to_pylist())) == picked
        _check(schema, datas, [("label", "eq", b"host-1")], window_ms=window, model_input=(plain, labelled, []))


@pytest.mark.parametrize("codec", [ParquetCompression.Uncompressed, ParquetCompression.Snappy, ParquetCompression.Zstd])
@pytest.mark.parametrize("kind", ["plain", "delta_dict"])
def test_quantile_codecs_and_encodings(codec, kind):
    rng = np.random.default_rng(31)
    schema = _schema(value_t=pa.int64())
    cols = _gauge_cols(rng, [70] * 8 + [900], ints=True, null_p=0.03)
    if kind == "plain":
        cfg = WriteConfig(compression=codec, max_row_group_size=150)
    else:
        cfg = WriteConfig(compression=codec, max_row_group_size=150,
                          column_options={"ts": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                          "series_id": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                          "value": ColumnOptions(enable_dict=True)})
    _check(schema, [_write(schema, cols, 32, cfg)], window_ms=15_000)


# ----------------------------------------------------------------------------------------------------------- refusals, empty results
def test_quantile_refusals_before_device_work():
    rng = np.random.default_rng(71)
    schema = _schema(extra=[pa.field("blob", pa.binary()), pa.field("fval", pa.float32())])
    cols = _gauge_cols(rng, [10] * 3)
    cols["blob"] = [b"x"] * len(cols["ts"])
    cols["fval"] = [1.0] * len(cols["ts"])
    data = _write(schema, cols, 70)
    handle = SchemaHandle(schema.arrow_schema, 2)
    append = StorageSchema.try_new(pa.schema([pa.field("series_id", pa.uint64()), pa.field("ts", pa.int64()), pa.field("blob", pa.binary())]), 2,
                                   UpdateMode.Append)                     # every value column of an Append table is Binary
    handle_a = SchemaHandle(append.arrow_schema, 2, UpdateMode.Append)
    eng = Engine(device=0)
    ins = _inputs([data])
    eng.scan_quantile_aggregate(handle, ins)
    before = eng.stats()
    assert before["kernel_launches"] > 0
    nan = float("nan")
    BINARY = "Binary columns cannot be grouped or aggregated"
    cases = [(handle, dict(quantiles=()), 1, "a quantile aggregate takes 1 to 16 quantiles"),
             (handle, dict(quantiles=(0.5,) * 17), 1, "a quantile aggregate takes 1 to 16 quantiles"),
             (handle, dict(quantiles=(0.5, nan)), 1, "a quantile must lie in [0, 1]"),
             (handle, dict(quantiles=(-0.01,)), 1, "a quantile must lie in [0, 1]"),
             (handle, dict(quantiles=(1.5,)), 1, "a quantile must lie in [0, 1]"),
             (handle, dict(value_col=-1), 1, "a quantile aggregate needs a value column"),
             (handle, dict(value_col=4), 1, BINARY),  # Binary value column
             (handle, dict(group_col=4), 1, BINARY),  # Binary group column
             (handle, dict(ts_col=4), 1, BINARY),  # Binary time column
             (handle, dict(ts_col=5, window_ms=1000), 1, "time column must be an integer column"),  # a float time column with buckets
             (handle, dict(mode=2), 1, "aggregation mode"),
             (handle, dict(value_col=40), 1, "aggregation column out of range"),
             (handle_a, dict(value_col=2), 1, BINARY),
             (handle_a, dict(value_col=1), 2, "aggregation over an Append-mode (BytesMergeOperator) table")]
    for h, kw, code, msg in cases:
        with pytest.raises(HgError) as ei:
            eng.scan_quantile_aggregate(h, ins, **kw)
        assert ei.value.code == code and eng._L.hg_last_error().decode() == msg, (kw, str(ei.value))
        assert eng.stats() == before, kw                 # refused before the call started: the last call's statistics are untouched
        if "quantiles" in kw or kw.get("value_col") == -1:
            continue
        # the spec's own checks: hg_scan_aggregate[_device] make them too, before the call
        for call in (eng.scan_aggregate, eng.scan_aggregate_device):
            with pytest.raises(HgError) as ei:
                call(h, ins, **{"value_col": 2, **kw})
            assert ei.value.code == code and eng._L.hg_last_error().decode() == msg, (call.__name__, kw, str(ei.value))
            assert eng.stats() == before, (call.__name__, kw)
    # an Append-mode table is refused without any SST too, by every call that takes this spec
    for call in (eng.scan_quantile_aggregate, eng.scan_aggregate, eng.scan_aggregate_device):
        with pytest.raises(HgError) as ei:
            call(handle_a, [], value_col=1)
        assert ei.value.code == 2 and "Append" in str(ei.value), call.__name__
        assert eng.stats() == before, call.__name__
    # a null quantile pointer, through the C entry point
    from horaedb_b200._ffi import ArrowArrayStream, HgAggSpec, lib
    import ctypes as C
    spec = HgAggSpec(0, -1, 0, 2, 0)
    stream = ArrowArrayStream()
    arr, keep = eng._descs(ins)
    rc = lib().hg_scan_quantile_aggregate(eng._h, C.byref(handle.desc), arr, C.c_size_t(1), None, C.c_size_t(0), C.byref(spec), None,
                                          C.c_uint32(1), C.byref(stream))
    assert rc == 1 and b"null quantiles" in lib().hg_last_error()
    assert eng.stats() == before
    eng.close()


def test_quantile_empty_input_and_no_passing_row():
    schema = _schema()
    rng = np.random.default_rng(81)
    data = _write(schema, _gauge_cols(rng, [10] * 3), 80)
    for window, group_col in ((0, 0), (60_000, 0), (0, -1), (60_000, -1)):
        want = (["series_id"] if group_col == 0 else []) + (["bucket"] if window else []) + ["count", "quantile_0", "quantile_1"]
        for datas, preds in (([], []), ([data], [("ts", "lt", T0 - 1)])):
            got, st, _ = _run(schema, datas, preds, ts_col=1, window_ms=window, group_col=group_col, quantiles=(0.5, 0.9))
            assert got.num_rows == 0 and got.column_names == want
            assert [got.schema.field(n).type for n in got.column_names[-3:]] == [pa.uint64(), pa.float64(), pa.float64()]
            assert st["groups_out"] == 0 and st["bytes_d2h"] == 0
            _assert_same(got, quantile_aggregate(datas, schema.arrow_schema, 2, preds, group_col=group_col, ts_col=1, window_ms=window,
                                                 quantiles=(0.5, 0.9)))


def test_quantile_bytes_d2h():
    schema = _schema()
    rng = np.random.default_rng(91)
    cols = _gauge_cols(rng, [20] * 5, null_p=0.1)
    cols["value"][:20] = [None] * 20
    got, st, _ = _run(schema, [_write(schema, cols, 90)], ts_col=1, window_ms=5_000, quantiles=(0.1, 0.5, 0.9))
    g = got.num_rows
    assert st["groups_out"] == g > 0 and got["quantile_0"].null_count > 0
    assert st["bytes_d2h"] == g * 8 * (3 + 3) + (g + 7) // 8          # key, bucket, count, 3 quantiles + one validity bitmap
