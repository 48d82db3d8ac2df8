"""Aggregates by label group (`hg_scan_aggregate_by_map`, `hg_scan_aggregate_by_map_device`, `hg_scan_quantile_aggregate_by_map`): the
caller's series -> group map decides every row's group (group_map_kernel), the map's keys filter and prune as an IN_SET predicate would.

Every case is compared bit for bit (a NaN matches any NaN) with two references:
  1. tests/group_map_model.py over the C oracle's deduplicated stream;
  2. the library itself: the same rows written with one more column grp = map[series] (u32), aggregated with `scan_aggregate` /
     `scan_quantile_aggregate` in HASH mode on grp, with `key IN_SET map.keys` as the last predicate, under HG_FLAG_NO_FUSED.  With the
     key column renamed to "group" the two tables must be equal column for column."""
import numpy as np
import pyarrow as pa
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_FUSED, HG_FLAG_NO_PRUNING, Engine, HgError, SchemaHandle, SstInput
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode
from group_map_model import aggregate_by_map, quantile_aggregate_by_map

pytestmark = pytest.mark.gpu
_ids = iter(range(170_000_000, 180_000_000))
T0 = sstgen.T0_MS
Q4 = (0.0, 0.5, 0.9, 1.0)
INT_TYPES = [pa.uint8(), pa.int8(), pa.uint16(), pa.int16(), pa.uint32(), pa.int32(), pa.uint64(), pa.int64()]
PK_TYPES = {"uint8", "int8", "uint32", "int32", "uint64", "int64"}       # the types a primary key may have


def _schema(key_t=pa.uint64(), value_t=pa.float64(), pk=("series_id", "ts"), extra=()):
    """series_id, ts, value, tag (u32), grp (u32: the map's group, for the in-library reference), *extra; pk = the primary keys (in
    front, in this order)"""
    fields = {"series_id": pa.field("series_id", key_t), "ts": pa.field("ts", pa.int64()), "value": pa.field("value", value_t),
              "tag": pa.field("tag", pa.uint32()), "grp": pa.field("grp", pa.uint32())}
    for f in extra:
        fields[f.name] = f
    order = list(pk) + [n for n in fields if n not in pk]
    user = pa.schema([fields[n] for n in order])
    s = StorageSchema.try_new(user, len(pk), UpdateMode.Overwrite)
    s.user = user
    s.num_pk = len(pk)
    return s


def _write(schema, cols, seq, cfg=None):
    batch = pa.RecordBatch.from_arrays([pa.array(cols[f.name], f.type) for f in schema.user], schema=schema.user)
    return sstgen.write_sst(schema, batch, seq=seq, cfg=cfg or WriteConfig(max_row_group_size=500))


def _cols(rng, sids, n_per, t0=T0, step=1000, null_p=0.05, n_tags=4):
    sid, ts, val, tag = [], [], [], []
    for s in sids:
        sid += [s] * n_per
        ts += [t0 + p * step for p in range(n_per)]
        v = rng.normal(50.0, 20.0, n_per)
        val += [None if rng.random() < null_p else float(x) for x in v]
        tag += rng.integers(0, n_tags, n_per).tolist()
    return {"series_id": sid, "ts": ts, "value": val, "tag": tag}


def _with_grp(cols, key, lookup):
    """cols plus grp = lookup[key] (0 for a key outside the map: such rows are filtered out either way)"""
    out = dict(cols)
    out["grp"] = [lookup.get(k, 0) if k is not None else 0 for k in cols[key]]
    return out


def _lookup(schema, key, keys, groups):
    from group_map_model import map_lookup
    return map_lookup(schema.arrow_schema.field(key).type, keys, groups)


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


def _f64_bits(col):
    a = col.fill_null(0.0).to_numpy().astype(np.float64)
    bits = a.view(np.uint64).copy()
    bits[np.isnan(a)] = 0x7FF8000000000000
    return bits.tolist()


def _assert_same(got, exp):
    assert got.column_names == exp.column_names, (got.column_names, exp.column_names)
    assert got.num_rows == exp.num_rows, (got.num_rows, exp.num_rows)
    for name in exp.column_names:
        g, e = got[name].combine_chunks(), exp[name].combine_chunks()
        assert g.type == e.type, (name, g.type, e.type)
        assert g.is_valid().to_pylist() == e.is_valid().to_pylist(), name
        if e.type == pa.float64():
            assert _f64_bits(g) == _f64_bits(e), name
        else:
            assert g.to_pylist() == e.to_pylist(), name


def _renamed(t, key_name):
    return t.rename_columns(["group" if n == key_name else n for n in t.column_names])


def _run(schema, datas, keys, groups, preds=(), flags=0, resident=False, quantiles=None, key="series_id", **kw):
    """(by-map table, its stats, the in-library reference table)"""
    handle = SchemaHandle(schema.arrow_schema, schema.num_pk)
    eng, ins = _engine(handle, datas, flags, resident)
    names = schema.arrow_schema.names
    kc, gc = names.index(key), names.index("grp")
    ref_preds = [*preds, (key, "in_set", np.asarray(keys))]
    if quantiles is None:
        got = eng.scan_aggregate_by_map(handle, ins, keys, groups, preds, group_col=kc, **kw)
        st = eng.stats()
        eng.set_flags(flags | HG_FLAG_NO_FUSED)
        ref = eng.scan_aggregate(handle, ins, ref_preds, group_col=gc, **{**kw, "mode": HG_AGG_HASH})
    else:
        got = eng.scan_quantile_aggregate_by_map(handle, ins, keys, groups, preds, group_col=kc, quantiles=quantiles, **kw)
        st = eng.stats()
        eng.set_flags(flags | HG_FLAG_NO_FUSED)
        ref = eng.scan_quantile_aggregate(handle, ins, ref_preds, group_col=gc, quantiles=quantiles, **{**kw, "mode": HG_AGG_HASH})
    eng.close()
    return got, st, _renamed(ref, "grp")


def _check(schema, datas, keys, groups, preds=(), oracle_preds=None, modes=(HG_AGG_HASH,), quantiles=None, transient_only=False,
           key="series_id", ts_col=1, window_ms=0, value_col=2, model_keys=None, model_input=None):
    """the by-map table == the model's == the in-library reference; transient and resident, with and without pruning, in every mode.
    model_keys: (keys, groups) the model reads instead (a subset holding every key the data has); model_input: (schema, datas) the model
    reads instead (the C oracle has no Binary columns)"""
    names = schema.arrow_schema.names
    kc = names.index(key)
    ts_col = names.index("ts") if ts_col == 1 else ts_col
    value_col = names.index("value") if value_col == 2 else value_col
    mk, mg = model_keys or (keys, groups)
    m_preds = list(oracle_preds if oracle_preds is not None else preds)
    m_schema, m_datas = model_input or (schema, datas)
    if quantiles is None:
        exp = aggregate_by_map(m_datas, m_schema.arrow_schema, m_schema.num_pk, m_preds, kc, mk, mg, ts_col, window_ms, value_col)
    else:
        exp = quantile_aggregate_by_map(m_datas, m_schema.arrow_schema, m_schema.num_pk, m_preds, kc, mk, mg, ts_col, window_ms, value_col,
                                        quantiles)
    runs = ((0, False),) if transient_only else ((0, False), (0, True), (HG_FLAG_NO_PRUNING, False))
    for mode in modes:
        for flags, resident in runs:
            got, st, ref = _run(schema, datas, keys, groups, preds, flags=flags, resident=resident, quantiles=quantiles, key=key,
                                ts_col=ts_col, window_ms=window_ms, value_col=value_col, mode=mode)
            _assert_same(got, exp)
            _assert_same(got, ref)
            assert st["path"] == 0 and st["groups_out"] == got.num_rows
    return exp


def _map(rng, sids, n_groups, extra=0, lo=10_000_000):
    """every series of sids into one of n_groups ordinals, plus `extra` keys that no row has"""
    keys = np.array(list(sids) + list(rng.choice(np.arange(lo, lo + 10 * extra + 1), extra, replace=False)), dtype=np.int64)
    groups = rng.integers(0, n_groups, len(keys)).astype(np.uint32)
    return keys, groups


# ----------------------------------------------------------------------------------------------------------------- windows, modes
@pytest.mark.parametrize("window_ms", [0, 7_000, 60_000])
def test_by_map_windows_and_modes(window_ms):
    """negative timestamps, RUNS and HASH equal; half the series mapped, into 3 groups, with keys no row has"""
    rng = np.random.default_rng(window_ms)
    schema = _schema(key_t=pa.int64())
    sids = list(range(-6, 14))
    keys, groups = _map(rng, sids[::2], 3, extra=5)
    lk = _lookup(schema, "series_id", keys, groups)
    cols = _with_grp(_cols(rng, sids, 60, t0=-45_000), "series_id", lk)
    exp = _check(schema, [_write(schema, cols, 3)], keys, groups, window_ms=window_ms, modes=(HG_AGG_RUNS, HG_AGG_HASH))
    assert exp.num_rows > 0 and set(exp["group"].to_pylist()) <= set(groups.tolist())


def test_by_map_count_only_and_quantiles_share_groups():
    rng = np.random.default_rng(2)
    schema = _schema()
    sids = list(range(40))
    keys, groups = _map(rng, sids, 5)
    cols = _with_grp(_cols(rng, sids, 30), "series_id", _lookup(schema, "series_id", keys, groups))
    datas = [_write(schema, cols, 4)]
    cnt = _check(schema, datas, keys, groups, value_col=-1, window_ms=10_000)
    assert cnt.column_names == ["group", "bucket", "count"]
    q = _check(schema, datas, keys, groups, window_ms=10_000, quantiles=Q4)
    assert q["group"].to_pylist() == cnt["group"].to_pylist() and q["count"].to_pylist() == cnt["count"].to_pylist()


# ----------------------------------------------------------------------------------------------------------------------- maps
def test_by_map_empty_map():
    """an empty map matches no row: a zero-row stream with the full schema, for every call"""
    rng = np.random.default_rng(3)
    schema = _schema()
    cols = _with_grp(_cols(rng, range(5), 20), "series_id", {})
    datas = [_write(schema, cols, 5)]
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    for window in (0, 60_000):
        got = eng.scan_aggregate_by_map(handle, _inputs(datas), np.array([], np.uint64), np.array([], np.uint32), group_col=0, ts_col=1,
                                        window_ms=window, value_col=2)
        assert got.num_rows == 0 and got.column_names == ["group"] + (["bucket"] if window else []) + ["count", "sum", "min", "max"]
        assert got.schema.field("group").type == pa.uint32()
        assert eng.stats()["groups_out"] == 0 and eng.stats()["rows_out"] == 0
        q = eng.scan_quantile_aggregate_by_map(handle, _inputs(datas), [], [], group_col=0, ts_col=1, window_ms=window, quantiles=(0.5,))
        assert q.num_rows == 0 and q.column_names[-2:] == ["count", "quantile_0"]
    eng.close()
    _check(schema, datas, np.array([], np.uint64), np.array([], np.uint32), window_ms=60_000)


def test_by_map_one_key():
    rng = np.random.default_rng(4)
    schema = _schema()
    cols = _with_grp(_cols(rng, range(30), 25), "series_id", {17: 9})
    exp = _check(schema, [_write(schema, cols, 6)], [17], [9], window_ms=7_000)
    assert set(exp["group"].to_pylist()) == {9} and sum(exp["count"].to_pylist()) == 25


def test_by_map_unsorted_with_duplicates_equals_sorted():
    rng = np.random.default_rng(5)
    schema = _schema()
    sids = list(range(50))
    keys, groups = _map(rng, sids, 7, extra=20)
    order = np.argsort(keys, kind="stable")
    skeys, sgroups = keys[order], groups[order]
    dup = rng.integers(0, len(keys), 40)
    ukeys = np.concatenate([keys, keys[dup]])
    ugroups = np.concatenate([groups, groups[dup]])
    perm = rng.permutation(len(ukeys))
    ukeys, ugroups = ukeys[perm], ugroups[perm]
    cols = _with_grp(_cols(rng, sids, 20), "series_id", _lookup(schema, "series_id", keys, groups))
    datas = [_write(schema, cols, 7)]
    a = _check(schema, datas, skeys, sgroups, window_ms=60_000)
    b = _check(schema, datas, ukeys, ugroups, window_ms=60_000)
    _assert_same(b, a)


def test_by_map_of_16m_keys():
    """HG_MAX_IN_SET keys, unsorted, 1 000 of them present in the data"""
    rng = np.random.default_rng(6)
    schema = _schema()
    n = 1 << 24
    keys = rng.permutation(np.arange(1, 3 * n, 3, dtype=np.uint64)[:n])
    groups = (keys % 1000).astype(np.uint32)
    present = keys[:1000]
    sids = sorted(int(x) for x in present[::10]) + [2, 5]                   # 2 and 5 are no key (keys are 1 mod 3)
    cols = _cols(rng, sids, 12)
    lk = {int(k): int(g) for k, g in zip(present, groups[:1000])}
    cols = _with_grp(cols, "series_id", lk)
    exp = _check(schema, [_write(schema, cols, 8)], keys, groups, window_ms=0, transient_only=True, model_keys=(present, groups[:1000]))
    assert sum(exp["count"].to_pylist()) == 12 * (len(sids) - 2)


def test_by_map_ordinal_extremes_and_sparse_ordinals():
    """ordinals 0 and 0xFFFFFFFF order as unsigned; sparse ordinals stay as given"""
    rng = np.random.default_rng(7)
    schema = _schema()
    sids = list(range(12))
    groups = np.array([0xFFFFFFFF, 0, 1 << 31, 7, 0xFFFFFFFF, 0, 123456789, 1 << 31, 5, 5, 0x80000001, 42], dtype=np.uint32)
    cols = _with_grp(_cols(rng, sids, 15), "series_id", dict(zip(sids, groups.tolist())))
    exp = _check(schema, [_write(schema, cols, 9)], np.array(sids), groups, window_ms=0)
    assert exp["group"].to_pylist() == sorted(set(groups.tolist()))


# -------------------------------------------------------------------------------------------------------------------- key columns
@pytest.mark.parametrize("key_t", INT_TYPES, ids=str)
def test_by_map_key_types_at_their_limits(key_t):
    """keys at the type's minimum and maximum; keys outside a narrow column's range never match.  Primary-key types are pk0, u16 / i16 a
    value column."""
    rng = np.random.default_rng(key_t.bit_width)
    info = np.iinfo(key_t.to_pandas_dtype())
    lo, hi = int(info.min), int(info.max)
    vals = sorted({lo, lo + 1, -1 if lo < 0 else 2, 0, 1, hi - 1, hi})
    pk = ("series_id", "ts") if str(key_t) in PK_TYPES else ("ts",)
    schema = _schema(key_t=key_t, pk=pk)
    n_per = 9
    cols = _cols(rng, vals, n_per)
    if len(pk) == 1:                                                      # one primary key: distinct timestamps for every row
        cols["ts"] = [T0 + i for i in range(len(cols["ts"]))]
    keys = sorted({lo, hi, 0, -1 if lo < 0 else 2})
    wide = [k & 0xFFFFFFFFFFFFFFFF for k in keys]
    if key_t.bit_width < 64:                                              # widened keys the column cannot hold
        wide += sorted({k & 0xFFFFFFFFFFFFFFFF for k in (lo - 1, hi + 1, -(1 << 63), (1 << 63) - 1, (1 << 64) - 1)} - set(wide))
    groups = np.arange(len(wide), dtype=np.uint32)[::-1].copy()
    cols = _with_grp(cols, "series_id", _lookup(schema, "series_id", np.array(wide, dtype=np.uint64), groups))
    datas = [_write(schema, cols, 10)]
    wide = np.array(wide, dtype=np.uint64)
    exp = _check(schema, datas, wide, groups, key="series_id", window_ms=30_000)
    assert sum(exp["count"].to_pylist()) == n_per * len(keys)


def test_by_map_on_the_second_primary_key():
    """a (metric_id, tsid, ...) table: the map's keys are the tsid, pk1, under a metric_id predicate"""
    rng = np.random.default_rng(11)
    schema = _schema(pk=("metric", "series_id"), extra=[pa.field("metric", pa.uint32())])
    cols = {"metric": [], "series_id": [], "ts": [], "value": [], "tag": []}
    for m in range(3):
        for s in range(25):
            n = 8
            cols["metric"] += [m] * n
            cols["series_id"] += [1000 * m + s] * n
            cols["ts"] += [T0 + 1000 * p for p in range(n)]
            cols["value"] += [float(x) for x in rng.normal(0, 10, n)]
            cols["tag"] += [0] * n
    keys = np.array([1000 * m + s for m in range(3) for s in range(0, 25, 2)], dtype=np.uint64)
    groups = (keys % 4).astype(np.uint32)
    cols = _with_grp(cols, "series_id", _lookup(schema, "series_id", keys, groups))
    datas = [_write(schema, cols, 12)]
    # (ts is a value column here: no buckets in this schema's first two columns)
    _check(schema, datas, keys, groups, preds=[("metric", "eq", 1)], window_ms=0)
    _check(schema, datas, keys, groups, window_ms=5_000)


def test_by_map_on_a_value_column_with_nulls():
    """the map's key column is `tag` (u32, NULL in places): NULL keys never match"""
    rng = np.random.default_rng(12)
    schema = _schema()
    cols = _cols(rng, range(20), 30, n_tags=6)
    cols["tag"] = [None if i % 7 == 0 else t for i, t in enumerate(cols["tag"])]
    keys, groups = np.array([0, 2, 3, 5, 99], dtype=np.uint64), np.array([1, 1, 0, 2, 3], dtype=np.uint32)
    cols = _with_grp(cols, "tag", _lookup(schema, "tag", keys, groups))
    _check(schema, [_write(schema, cols, 13)], keys, groups, key="tag", window_ms=60_000, modes=(HG_AGG_RUNS, HG_AGG_HASH))


# ------------------------------------------------------------------------------------------------------------------------ inputs
@pytest.mark.parametrize("codec", [ParquetCompression.Uncompressed, ParquetCompression.Snappy, ParquetCompression.Zstd])
@pytest.mark.parametrize("kind", ["plain", "delta_dict"])
def test_by_map_codecs_and_encodings(codec, kind):
    rng = np.random.default_rng(21)
    schema = _schema()
    sids = list(range(30))
    keys, groups = _map(rng, sids[1::3] + sids[::5], 4)
    keys = np.unique(keys)
    groups = groups[: len(keys)]
    cols = _with_grp(_cols(rng, sids, 40), "series_id", _lookup(schema, "series_id", keys, groups))
    if kind == "plain":
        cfg = WriteConfig(compression=codec, max_row_group_size=150)
    else:
        cfg = WriteConfig(compression=codec, max_row_group_size=150,
                          column_options={"ts": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                          "series_id": ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked),
                                          "value": ColumnOptions(enable_dict=True)})
    _check(schema, [_write(schema, cols, 22, cfg)], keys, groups, window_ms=15_000)


def test_by_map_dedups_before_grouping():
    """a newer SST overwrites rows of an older one (the value, and a NULL): only the newest versions are grouped"""
    schema = _schema()
    keys, groups = np.array([1, 2, 3], dtype=np.uint64), np.array([0, 1, 0], dtype=np.uint32)
    lk = dict(zip([1, 2, 3], [0, 1, 0]))
    old = _with_grp({"series_id": [1] * 4 + [2] * 3 + [3] * 2, "ts": [T0 + i for i in range(4)] + [T0, T0 + 1, T0 + 2] + [T0, T0 + 1],
                     "value": [1.0, 2.0, 1e9, 4.0, 7.0, -1e9, 9.0, 3.0, 3.5], "tag": [0] * 9}, "series_id", lk)
    new = _with_grp({"series_id": [1, 2, 4], "ts": [T0 + 2, T0 + 1, T0], "value": [3.0, None, 8.0], "tag": [1, 1, 1]}, "series_id", lk)
    exp = _check(schema, [_write(schema, old, 30), _write(schema, new, 31)], keys, groups, window_ms=0)
    assert exp["count"].to_pylist() == [6, 3] and exp["max"].to_pylist() == [4.0, 9.0]


# -------------------------------------------------------------------------------------------------------------------- predicates
def test_by_map_with_caller_predicates():
    """a time range, `tag =`, a Binary predicate and an IN_SET on another column, before the map's set"""
    rng = np.random.default_rng(41)
    schema = _schema(extra=[pa.field("label", pa.binary())])
    sids = list(range(1000, 1040))
    keys, groups = _map(rng, sids[::2], 5, extra=1000)
    cols = _cols(rng, sids, 50)
    cols["label"] = [b"host-%d" % (i % 3) for i in range(len(cols["ts"]))]
    cols = _with_grp(cols, "series_id", _lookup(schema, "series_id", keys, groups))
    datas = [_write(schema, cols, 40, WriteConfig(max_row_group_size=200))]
    # the model reads the same rows without the Binary column (the C oracle has none)
    plain = _schema()
    names = plain.arrow_schema.names[:-2]
    whole = (plain, [_write(plain, {k: cols[k] for k in names}, 40)])
    ts_range = [("ts", "ge", T0 + 12_000), ("ts", "lt", T0 + 37_000)]
    for window in (0, 10_000):
        _check(schema, datas, keys, groups, ts_range, window_ms=window, model_input=whole)
        _check(schema, datas, keys, groups, [("tag", "eq", 2), *ts_range], window_ms=window, model_input=whole)
        _check(schema, datas, keys, groups, [("tag", "in_set", np.array([0, 3, 77], np.uint32))], window_ms=window, model_input=whole,
               oracle_preds=[("tag", "in", [0, 3, 77])])
    # the Binary predicate: the model reads the rows it keeps (one file, no older versions)
    keep = [i for i, x in enumerate(cols["label"]) if x == b"host-1"]
    labelled = [_write(plain, {k: [cols[k][i] for i in keep] for k in names}, 40)]
    exp = aggregate_by_map(labelled, plain.arrow_schema, 2, [], 0, keys, groups, 1, 10_000, 2)
    for flags in (0, HG_FLAG_NO_PRUNING):
        got, _, ref = _run(schema, datas, keys, groups, [("label", "eq", b"host-1")], flags=flags, ts_col=1, window_ms=10_000, value_col=2)
        _assert_same(got, exp)
        _assert_same(got, ref)


def test_by_map_seven_predicates_accepted_eight_refused():
    rng = np.random.default_rng(42)
    schema = _schema()
    cols = _with_grp(_cols(rng, range(10), 40), "series_id", {s: s % 2 for s in range(10)})
    datas = [_write(schema, cols, 41)]
    keys, groups = np.arange(10), np.arange(10) % 2
    seven = [("ts", "ge", T0), ("ts", "lt", T0 + 30_000), ("tag", "le", 2), ("tag", "ne", 1), ("series_id", "ge", 1),
             ("series_id", "lt", 9), ("value", "gt", -1e9)]
    _check(schema, datas, keys, groups, seven, window_ms=10_000)
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    with pytest.raises(HgError) as ei:
        eng.scan_aggregate_by_map(handle, _inputs(datas), keys, groups, seven + [("tag", "ge", 0)], group_col=0, value_col=2)
    assert ei.value.code == 2 and "more than 8 predicates" in str(ei.value)
    eng.close()


def test_by_map_prunes_row_groups():
    """a map of a few series decodes fewer rows than the same call without pruning; the same on transient inputs"""
    rng = np.random.default_rng(43)
    schema = _schema()
    sids = list(range(200))
    keys, groups = np.array([3, 4, 150], dtype=np.uint64), np.array([0, 1, 0], dtype=np.uint32)
    cols = _with_grp(_cols(rng, sids, 50), "series_id", _lookup(schema, "series_id", keys, groups))
    datas = [_write(schema, cols, 42, WriteConfig(max_row_group_size=400))]
    _check(schema, datas, keys, groups, window_ms=60_000)
    decoded, h2d = {}, {}
    for flags in (0, HG_FLAG_NO_PRUNING):
        for resident in (False, True):
            _, st, _ = _run(schema, datas, keys, groups, flags=flags, resident=resident, ts_col=1, window_ms=60_000, value_col=2)
            decoded[flags, resident], h2d[flags, resident] = st["rows_decoded"], st["bytes_h2d"]
            assert st["rows_filtered"] == 150
    assert decoded[0, True] < decoded[HG_FLAG_NO_PRUNING, True] == 10_000
    assert decoded[0, False] < decoded[HG_FLAG_NO_PRUNING, False] and h2d[0, False] < h2d[HG_FLAG_NO_PRUNING, False]


def test_by_map_stats_count_the_map_upload():
    """on resident inputs bytes_h2d = the IN_SET call's (the keys) + 4 bytes per group ordinal"""
    rng = np.random.default_rng(44)
    schema = _schema()
    keys, groups = np.arange(0, 60, 2, dtype=np.uint64), (np.arange(30) % 3).astype(np.uint32)
    cols = _with_grp(_cols(rng, range(60), 20), "series_id", _lookup(schema, "series_id", keys, groups))
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng, ins = _engine(handle, [_write(schema, cols, 43)], HG_FLAG_NO_FUSED, True)
    eng.scan_aggregate_by_map(handle, ins, keys, groups, group_col=0, value_col=2)
    st = eng.stats()
    eng.scan_aggregate(handle, ins, [("series_id", "in_set", keys)], group_col=0, value_col=2, mode=HG_AGG_HASH)
    st_in = eng.stats()
    eng.close()
    assert st["bytes_h2d"] == st_in["bytes_h2d"] + 4 * len(keys)
    assert st["rows_filtered"] == st_in["rows_filtered"] == 600 and st["groups_out"] == 3


# ------------------------------------------------------------------------------------------------------------------------- quantiles
def test_by_map_quantiles_across_the_tiers():
    """small series merged into groups of every tier: <= 32 values, <= 4 096 and larger, one above 16 384 (several blocks a pass)"""
    rng = np.random.default_rng(51)
    schema = _schema()
    parts = [(range(0, 20), 1, 9), (range(20, 23), 10, 11), (range(23, 24), 70, 7), (range(24, 124), 70, 2), (range(124, 404), 70, 3)]
    cols = {"series_id": [], "ts": [], "value": [], "tag": []}
    lk = {}
    for sids, n_per, g in parts:
        c = _cols(rng, sids, n_per, step=1, null_p=0.1)
        for k in cols:
            cols[k] += c[k]
        lk.update({s: g for s in sids})
    keys = np.arange(404, dtype=np.uint64)
    groups = np.array([lk[s] for s in range(404)], np.uint32)
    cols = _with_grp(cols, "series_id", lk)
    datas = [_write(schema, cols, 50, WriteConfig(max_row_group_size=5000))]
    exp = _check(schema, datas, keys, groups, quantiles=(0.0, 0.01, 0.5, 0.99, 1.0), transient_only=True, window_ms=0)
    counts = dict(zip(exp["group"].to_pylist(), exp["count"].to_pylist()))
    assert counts == {9: 20, 11: 30, 7: 70, 2: 7000, 3: 19_600}
    _check(schema, datas, keys, groups, quantiles=(0.5, 0.9, 0.99), transient_only=True, window_ms=7_000, modes=(HG_AGG_RUNS, HG_AGG_HASH))


# ------------------------------------------------------------------------------------------------------------------- device results
def test_aggregate_device_result_by_map_packs_and_reduces():
    """scan_aggregate_by_map_device + export_packed == the stream (ordinals zero-extended); a world-1 REDUCE combine == the model"""
    import torch
    from horaedb_b200._ffi import HG_COMBINE_REDUCE, DeviceArray
    from group_map_model import reduce_shards
    rng = np.random.default_rng(61)
    schema = _schema()
    sids = list(range(40))
    keys = np.arange(40, dtype=np.uint64)
    groups = np.where(np.arange(40) % 3 == 0, 0xFFFFFFFF, np.arange(40) % 5).astype(np.uint32)
    cols = _with_grp(_cols(rng, sids, 30), "series_id", dict(zip(sids, groups.tolist())))
    datas = [_write(schema, cols, 60)]
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    ins = _inputs(datas)
    kw = dict(group_col=0, ts_col=1, window_ms=10_000, value_col=2)
    table = eng.scan_aggregate_by_map(handle, ins, keys, groups, **kw)
    dev = eng.scan_aggregate_by_map_device(handle, ins, keys, groups, **kw)
    G = int(dev.num_groups)
    assert G == table.num_rows > 0
    gk = torch.as_tensor(DeviceArray(dev.d_gkey, G, "<u4"), device="cuda").cpu().numpy()
    assert gk.tolist() == table["group"].to_pylist()
    block = torch.full((6, G + 5), -1, dtype=torch.int64, device="cuda")
    eng.export_packed(block.data_ptr(), G + 5)
    torch.cuda.synchronize()
    hb = block.cpu().numpy()
    assert hb[0, :G].tolist() == table["group"].to_pylist()                   # zero-extended: 0xFFFFFFFF stays positive
    assert hb[1, :G].tolist() == table["bucket"].to_pylist() and hb[2, :G].tolist() == table["count"].to_pylist()
    for j, name in ((3, "sum"), (4, "min"), (5, "max")):
        assert hb[j, :G].tolist() == np.asarray(table[name].to_numpy(), np.float64).view(np.int64).tolist()
    assert not hb[:, G:].any()
    eng.comm_init(Engine.comm_unique_id(), 0, 1)
    eng.scan_aggregate_by_map_device(handle, ins, keys, groups, **kw)
    cmb = eng.combine(HG_COMBINE_REDUCE, 0)
    eng.comm_sync()
    n, cap = int(cmb.num_groups), int(cmb.reduced_capacity)
    tbl = torch.as_tensor(DeviceArray(cmb.d_reduced, 6 * cap, "<i8"), device="cuda").cpu().numpy().reshape(6, cap)[:, :n]
    acc = reduce_shards([aggregate_by_map(datas, schema.arrow_schema, 2, [], 0, keys, groups, 1, 10_000, 2)])
    ks = sorted(acc)
    assert n == len(ks)
    assert tbl[0].tolist() == [k[0] for k in ks] and tbl[1].tolist() == [k[1] for k in ks] and tbl[2].tolist() == [acc[k][0] for k in ks]
    for j in range(1, 4):
        assert tbl[2 + j].tolist() == np.array([acc[k][j] for k in ks], np.float64).view(np.int64).tolist()
    eng.comm_destroy()
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------- refusals
def test_by_map_refusals_before_device_work():
    import ctypes as C
    from horaedb_b200._ffi import ArrowArrayStream, HgAggDevice, HgAggSpec, HgGroupMap, lib
    rng = np.random.default_rng(71)
    schema = _schema(extra=[pa.field("blob", pa.binary()), pa.field("fval", pa.float32())])
    cols = _with_grp(_cols(rng, range(3), 10), "series_id", {})
    cols["blob"] = [b"x"] * len(cols["ts"])
    cols["fval"] = [1.0] * len(cols["ts"])
    names = schema.arrow_schema.names
    blob, fval = names.index("blob"), names.index("fval")
    data = _write(schema, cols, 70)
    handle = SchemaHandle(schema.arrow_schema, 2)
    append = StorageSchema.try_new(pa.schema([pa.field("series_id", pa.uint64()), pa.field("ts", pa.int64()), pa.field("blob", pa.binary())]), 2,
                                   UpdateMode.Append)
    handle_a = SchemaHandle(append.arrow_schema, 2, UpdateMode.Append)
    eng = Engine(device=0)
    ins = _inputs([data])
    keys, groups = np.array([0, 1, 2], np.uint64), np.array([0, 0, 1], np.uint32)
    eng.scan_aggregate_by_map(handle, ins, keys, groups, value_col=2)
    before = eng.stats()
    assert before["kernel_launches"] > 0
    agg_cases = [(handle, dict(keys=[1, 2, 1], groups=[0, 1, 1]), 1, "two different groups"),
                 (handle, dict(group_col=-1), 1, "key column"),
                 (handle, dict(group_col=blob, keys=[], groups=[]), 1, "Binary"),
                 (handle, dict(value_col=blob), 1, "Binary"),
                 (handle, dict(ts_col=blob), 1, "Binary"),
                 (handle, dict(ts_col=fval, window_ms=1000), 1, "integer"),
                 (handle, dict(mode=2), 1, "mode"),
                 (handle, dict(value_col=40), 1, "out of range"),
                 (handle, dict(group_col=fval, keys=[], groups=[]), 2, "float"),
                 (handle, dict(preds=[("tag", "ge", 0)] * 8), 2, "more than 8 predicates"),
                 (handle_a, dict(value_col=-1), 2, "Append")]
    for h, kw, code, msg in agg_cases:
        args = dict(keys=keys, groups=groups, group_col=0, value_col=2)
        args.update(kw)
        k, g = args.pop("keys"), args.pop("groups")
        preds = args.pop("preds", ())
        for call in ("stream", "device", "quantile") if args["value_col"] >= 0 else ("stream", "device"):
            with pytest.raises(HgError) as ei:
                if call == "stream":
                    eng.scan_aggregate_by_map(h, ins, k, g, preds, **args)
                elif call == "device":
                    eng.scan_aggregate_by_map_device(h, ins, k, g, preds, **args)
                else:
                    eng.scan_quantile_aggregate_by_map(h, ins, k, g, preds, quantiles=(0.5,), **args)
            assert ei.value.code == code and msg in str(ei.value), (call, kw, str(ei.value))
            assert eng.stats() == before, (call, kw)
    for kw, msg in ((dict(quantiles=()), "1 to 16"), (dict(quantiles=(1.5,)), "[0, 1]"), (dict(value_col=-1), "value column")):
        with pytest.raises(HgError) as ei:
            eng.scan_quantile_aggregate_by_map(handle, ins, keys, groups, **{"value_col": 2, **kw})
        assert ei.value.code == 1 and msg in str(ei.value), kw
        assert eng.stats() == before
    # an Append-mode table is refused without any SST too
    for call in (eng.scan_aggregate_by_map, eng.scan_aggregate_by_map_device, eng.scan_quantile_aggregate_by_map):
        with pytest.raises(HgError) as ei:
            call(handle_a, [], keys, groups, value_col=1)
        assert ei.value.code == 2 and "Append" in str(ei.value), call.__name__
        assert eng.stats() == before, call.__name__
    # through the C entry points: a null map, null keys / groups with a count, a count above HG_MAX_IN_SET
    L = lib()
    spec = HgAggSpec(0, -1, 0, 2, 0)
    arr, keep = eng._descs(ins)
    kbuf = (C.c_uint64 * 3)(0, 1, 2)
    gbuf = (C.c_uint32 * 3)(0, 0, 1)
    maps = [(None, "null group map"),
            (HgGroupMap(None, gbuf, 3, 0), "null keys or groups"),
            (HgGroupMap(kbuf, None, 3, 0), "null keys or groups"),
            (HgGroupMap(kbuf, gbuf, (1 << 24) + 1, 0), "HG_MAX_IN_SET")]
    qs = (C.c_double * 1)(0.5)
    for m, msg in maps:
        mp = C.byref(m) if m is not None else None
        stream = ArrowArrayStream()
        out = HgAggDevice()
        for rc in (L.hg_scan_aggregate_by_map(eng._h, C.byref(handle.desc), arr, C.c_size_t(1), None, C.c_size_t(0), C.byref(spec), mp, C.byref(stream)),
                   L.hg_scan_aggregate_by_map_device(eng._h, C.byref(handle.desc), arr, C.c_size_t(1), None, C.c_size_t(0), C.byref(spec), mp, C.byref(out)),
                   L.hg_scan_quantile_aggregate_by_map(eng._h, C.byref(handle.desc), arr, C.c_size_t(1), None, C.c_size_t(0), C.byref(spec), mp,
                                                       qs, C.c_uint32(1), C.byref(stream))):
            assert rc == 1 and msg.encode() in L.hg_last_error(), (msg, L.hg_last_error())
            assert eng.stats() == before
    eng.close()
