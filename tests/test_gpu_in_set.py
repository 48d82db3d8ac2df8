"""Set-membership predicates (`HG_OP_IN_SET`, `("col", "in_set", values)`): `column IN (a set of up to 2^24 integers)`, evaluated by
eval_in_set_kernel on the general pipeline and used against chunk statistics to prune row groups.

Checked against the CPU oracle (whose `IN` has no length limit and defines the same semantics), against `HG_OP_IN` for lists it
accepts, and against a numpy model written here: keys are unique across the files of the large-set cases, so the expected rows are
the files' rows that `numpy.isin` keeps, in primary-key order.  The sizes come from the kernel's constants: a tile of rows is
searched in shared memory when its slice of the set has at most 4 096 keys (kInSetSmemKeys) and through splitters beyond."""
import ctypes as C
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from helpers import check_stream
from horaedb_b200 import sstgen
from horaedb_b200._ffi import (HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_FUSED, HG_FLAG_NO_PRUNING, Engine, HgError, HgPredicate, SchemaHandle, SstInput,
                               _check, lib)
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode
from oracle import oracle

pytestmark = pytest.mark.gpu
_ids = iter(range(140_000_000, 150_000_000))
SMEM_KEYS = 4096
INT_TYPES = [pa.uint8(), pa.int8(), pa.uint16(), pa.int16(), pa.uint32(), pa.int32(), pa.uint64(), pa.int64()]
T0 = sstgen.T0_MS


def _bounds(t):
    bits = t.bit_width
    return (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if pa.types.is_signed_integer(t) else (0, (1 << bits) - 1)


def _schema(key_t=pa.uint64(), tag_t=pa.uint32(), extra=()):
    user = pa.schema([pa.field("series_id", key_t), pa.field("ts", pa.int64()), pa.field("value", pa.float64()), pa.field("tag", tag_t), *extra])
    s = StorageSchema.try_new(user, 2)
    s.user = user
    return s


def _write(schema, cols, seq, cfg=None, sort=True):
    batch = pa.RecordBatch.from_arrays([pa.array(cols[f.name], f.type) for f in schema.user], schema=schema.user)
    return sstgen.write_sst(schema, batch, seq=seq, cfg=cfg or WriteConfig(max_row_group_size=1000), presorted=not sort)


def _inputs(datas):
    return [SstInput(id=next(_ids), data=d) for d in datas]


def _to_oracle(preds):
    return [(c, "in", [int(v) for v in lit]) if op == "in_set" else (c, op, lit) for c, op, lit in preds]


def _scan(schema, datas, preds, flags=0, resident=(), **kw):
    """batches of one scan and its statistics; files whose index is in `resident` are loaded first"""
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0, flags=flags)
    ins = _inputs(datas)
    for i in resident:
        eng.load_sst(handle, ins[i])
        ins[i] = SstInput(id=ins[i].id)
    got = list(eng.scan(handle, ins, preds, **kw))
    st = eng.stats()
    eng.close()
    return got, st


def _check_scan(schema, datas, preds, **kw):
    """IN_SET scan == the oracle's scan (batch boundaries included), with pruning and without, transient and resident"""
    exp = oracle.scan(datas, schema.arrow_schema, 2, _to_oracle(preds)).batches
    for flags, resident in ((0, ()), (HG_FLAG_NO_PRUNING, ()), (0, range(len(datas)))):
        got, st = _scan(schema, datas, preds, flags=flags, resident=resident, **kw)
        check_stream(got, exp)
        assert st["path"] & 1 == 0
    return exp


def _random_cols(rng, n, key_t, tag_t, key_lo=0, key_span=None, tag_null=0.0):
    lo, hi = _bounds(key_t)
    span = key_span or min(hi - lo, 5000)
    base = max(lo, key_lo)
    sid = np.sort(rng.integers(0, span, n)).astype(object) + base
    tlo, thi = _bounds(tag_t)
    tag = [int(x) for x in rng.integers(0, min(thi - tlo, 1 << 62), n)]
    tag = [None if rng.random() < tag_null else tlo + v for v in tag]
    return {"series_id": [int(x) for x in sid], "ts": (T0 + np.arange(n) * 1000).tolist(), "value": (rng.random(n) * 100 - 50).tolist(), "tag": tag}


# ------------------------------------------------------------------------------------------------- types, edges, shapes of the set
@pytest.mark.parametrize("tag_t", INT_TYPES, ids=str)
def test_in_set_every_integer_type_and_edge_literals(tag_t):
    """a value column of every integer type holding the type's edges; sets with the edges, unsorted with duplicates, sorted, empty, one
    value, every stored value, and values the file does not hold (literals outside the column's range included)"""
    rng = np.random.default_rng(tag_t.bit_width * 2 + pa.types.is_signed_integer(tag_t))
    schema = _schema(tag_t=tag_t)
    lo, hi = _bounds(tag_t)
    edges = sorted({lo, lo + 1, -1 if lo < 0 else 2, 0, 1, hi - 1, hi, (1 << 63) + 5 if hi > (1 << 63) else hi // 2})
    cols = _random_cols(rng, 3000, pa.uint64(), tag_t, tag_null=0.1)
    for i in range(0, 3000, 7):
        cols["tag"][i] = edges[(i // 7) % len(edges)]
    data = _write(schema, cols, 5)
    stored = sorted({v for v in cols["tag"] if v is not None})
    sets = [edges, [edges[-1], edges[0], edges[0], edges[-1], 0, 0], [], [edges[0]], stored, list(reversed(stored)) + stored[:5]]
    if tag_t.bit_width < 64:
        sets.append([hi + 1, lo - 1 if lo < 0 else hi + 300, hi])           # out-of-range literals match nothing
    for s in sets:
        exp = _check_scan(schema, [data], [("tag", "in_set", s)])
        keep = set(s)
        assert sum(b.num_rows for b in exp) == sum(v in keep for v in cols["tag"] if v is not None)
    absent = [v for v in range(max(lo, -300), min(hi, 300)) if v not in set(stored)][:40]
    assert sum(b.num_rows for b in _check_scan(schema, [data], [("tag", "in_set", absent)])) == 0


@pytest.mark.parametrize("key_t", [pa.uint8(), pa.int8(), pa.uint32(), pa.int32(), pa.uint64(), pa.int64()], ids=str)
def test_in_set_on_a_key_column_of_every_key_type(key_t):
    rng = np.random.default_rng(key_t.bit_width)
    schema = _schema(key_t=key_t)
    lo, hi = _bounds(key_t)
    cols = _random_cols(rng, 4000, key_t, pa.uint32(), key_lo=lo, key_span=min(hi - lo, 900))
    cols["series_id"][0], cols["series_id"][-1] = lo, hi
    if key_t == pa.uint64():
        cols["series_id"][-2] = (1 << 63) + 1
    data = _write(schema, cols, 6)
    ids = sorted(set(cols["series_id"]))
    picks = [ids[i] for i in rng.permutation(len(ids))[:len(ids) // 3]] + [lo, hi, ids[-2]]
    _check_scan(schema, [data], [("series_id", "in_set", picks)])
    _check_scan(schema, [data], [("series_id", "in_set", np.array(sorted(set(picks)), dtype=np.uint64 if lo == 0 else np.int64))])


# --------------------------------------------------------------------------------------------------------- sizes: the numpy model
def _big_files(nrows, id_span, seed, tag_span=1 << 31, rg=8192):
    """two files with disjoint, unique series ids spread over [0, id_span): every row its own series, so nothing is deduplicated"""
    rng = np.random.default_rng(seed)
    ids = np.sort(rng.choice(id_span, size=2 * nrows, replace=False).astype(np.uint64))
    schema = _schema()
    datas, tables = [], []
    for f in range(2):
        sid = ids[f * nrows:(f + 1) * nrows]
        cols = {"series_id": sid, "ts": T0 + np.arange(nrows, dtype=np.int64) * 10, "value": rng.random(nrows), "tag": rng.integers(0, tag_span, nrows).astype(np.uint32)}
        datas.append(_write(schema, cols, 20 + f, WriteConfig(max_row_group_size=rg), sort=False))
        tables.append(cols)
    return schema, datas, {k: np.concatenate([t[k] for t in tables]) for k in tables[0]}


def _check_big(schema, datas, allcols, col, values, extra=()):
    preds = [(col, "in_set", values), *extra]
    mask = np.isin(allcols[col], np.asarray(values).astype(allcols[col].dtype))
    for c, op, lit in extra:
        mask &= {"ge": allcols[c] >= lit, "lt": allcols[c] < lit, "ne": allcols[c] != lit}[op]
    for flags, resident in ((0, ()), (HG_FLAG_NO_PRUNING, (0, 1)), (0, (1,))):
        got, st = _scan(schema, datas, preds, flags=flags, resident=resident)
        t = pa.Table.from_batches(got, schema=pa.schema(list(schema.user))) if got else None
        assert (t.num_rows if t else 0) == int(mask.sum()) == st["rows_filtered"]
        if t:
            for name in ("series_id", "ts", "value", "tag"):
                assert np.array_equal(t[name].to_numpy(), allcols[name][mask]), name
        assert st["path"] & 1 == 0


SIZES = [1, 64, 65, SMEM_KEYS, SMEM_KEYS + 1, 100_000]


@pytest.mark.parametrize("size", SIZES)
def test_in_set_sizes_on_the_key_column(size):
    """a sorted key column: a tile spans few ids, so its slice of the set is short unless the set is dense"""
    schema, datas, allcols = _big_files(30_000, 200_000, 3)
    rng = np.random.default_rng(size)
    values = rng.choice(200_000, size=size, replace=False).astype(np.uint64)
    _check_big(schema, datas, allcols, "series_id", values)
    _check_big(schema, datas, allcols, "series_id", np.sort(values), extra=[("ts", "ge", T0 + 50_000), ("ts", "lt", T0 + 250_000)])


@pytest.mark.parametrize("size", SIZES)
def test_in_set_sizes_on_an_unsorted_value_column(size):
    """an unsorted column: every tile spans the whole range, its slice is the whole set — in shared memory up to 4 096 keys, through
    splitters from 4 097"""
    span = max(4 * size, 20_000)
    schema, datas, allcols = _big_files(30_000, 200_000, 4, tag_span=span)
    rng = np.random.default_rng(size + 1)
    values = (span // 4 + rng.choice(span // 2, size=min(size, span // 2), replace=False)).astype(np.uint32)
    _check_big(schema, datas, allcols, "tag", values)
    _check_big(schema, datas, allcols, "tag", values, extra=[("tag", "ne", int(values[0]))])


def test_in_set_million_values():
    """2^20 values: a dense set on the key column (long slices: splitters) and on the unsorted column"""
    schema, datas, allcols = _big_files(100_000, 2_000_000, 5, tag_span=4_000_000)
    rng = np.random.default_rng(11)
    _check_big(schema, datas, allcols, "series_id", rng.choice(2_000_000, size=1 << 20, replace=False).astype(np.uint64))
    _check_big(schema, datas, allcols, "tag", rng.choice(4_000_000, size=1 << 20, replace=False).astype(np.int64))


# ------------------------------------------------------------------------------------------------- IN_SET and IN are one predicate
def _overlapping(rng, schema, nfiles=3, n=5000, extra_cols=None, cfgs=None):
    datas = []
    for f in range(nfiles):
        cols = _random_cols(rng, n, pa.uint64(), pa.uint32(), key_span=300, tag_null=0.2 if f else 0.0)
        cols["ts"] = (T0 + rng.integers(0, 40, n) * 1000).tolist()                 # few timestamps per series: files share keys
        order = np.lexsort((cols["ts"], cols["series_id"]))
        keep = np.ones(n, bool)
        sk = [(cols["series_id"][i], cols["ts"][i]) for i in order]
        keep[1:] = [sk[i] != sk[i - 1] for i in range(1, n)]
        cols = {k: [v[i] for i, kp in zip(order, keep) if kp] for k, v in cols.items()}
        cols["tag"] = [None if v is None else v % 50 for v in cols["tag"]]
        if extra_cols:
            cols.update(extra_cols(rng, len(cols["ts"])))
        datas.append(_write(schema, cols, 30 + f, cfgs[f] if cfgs else WriteConfig(max_row_group_size=700), sort=False))
    return datas


@pytest.mark.parametrize("col,values", [("series_id", [5, 17, 250, 299, 5, 1000]), ("tag", list(range(0, 64))), ("tag", [7]), ("tag", [])])
@pytest.mark.parametrize("batch_size", [8192, 100])
def test_in_set_equals_in_for_short_lists(col, values, batch_size):
    """the same rows in the same batches as HG_OP_IN, over overlapping files: the filter runs before merge and dedup, so a set that
    hides the newest version of a key brings an older one back, exactly as IN does"""
    rng = np.random.default_rng(len(values))
    schema = _schema()
    datas = _overlapping(rng, schema)
    handle = SchemaHandle(schema.arrow_schema, 2)
    exp = oracle.scan(datas, schema.arrow_schema, 2, [(col, "in", values)], batch_size=batch_size).batches
    for resident in ((), (0, 2)):
        outs = []
        for op in ("in", "in_set"):
            eng = Engine(device=0, batch_size=batch_size)
            ins = _inputs(datas)
            for i in resident:
                eng.load_sst(handle, ins[i])
            outs.append(list(eng.scan(handle, ins, [(col, op, values)], keep_builtin=True)))
            st = eng.stats()
            eng.close()
        check_stream(outs[1], outs[0])
        check_stream([b.select(range(4)) for b in outs[1]], exp)
        assert st["path"] & 1 == 0


def test_in_set_hides_the_newest_version_of_a_key():
    schema = _schema()
    old = _write(schema, {"series_id": [1, 2], "ts": [T0, T0], "value": [1.0, 2.0], "tag": [10, 10]}, 1)
    new = _write(schema, {"series_id": [1, 2], "ts": [T0, T0], "value": [3.0, 4.0], "tag": [11, 10]}, 2)
    got, _ = _scan(schema, [old, new], [("tag", "in_set", [10])])
    t = pa.Table.from_batches(got)
    assert t["series_id"].to_pylist() == [1, 2] and t["value"].to_pylist() == [1.0, 4.0]
    _check_scan(schema, [old, new], [("tag", "in_set", [10])])


# -------------------------------------------------------------------------------------------------------------------- conjunctions
def test_in_set_conjunctions_nulls_and_aggregates():
    """IN_SET with a time range, a second IN_SET, `<>`; NULL-heavy and all-NULL chunks; RUNS and HASH aggregates with f64 sums bit for
    bit, on the general pipeline"""
    rng = np.random.default_rng(21)
    schema = _schema()
    datas = _overlapping(rng, schema)
    n = 1400
    cols = _random_cols(rng, n, pa.uint64(), pa.uint32(), key_span=300, tag_null=0.9)
    cols["tag"] = [None] * 700 + [None if v is None else v % 50 for v in cols["tag"][700:]]      # row group 0: all NULL
    datas.append(_write(schema, cols, 40, WriteConfig(max_row_group_size=700), sort=False))
    handle = SchemaHandle(schema.arrow_schema, 2)
    ids = rng.permutation(300)[:120].tolist()
    cases = [[("series_id", "in_set", ids), ("ts", "ge", T0 + 5000), ("ts", "lt", T0 + 30_000)],
             [("series_id", "in_set", ids), ("tag", "in_set", list(range(0, 50, 3)))],
             [("tag", "in_set", list(range(10, 40))), ("tag", "ne", 12), ("series_id", "ge", 40)],
             [("tag", "in_set", [1, 2, 3])]]
    for preds in cases:
        _check_scan(schema, datas, preds)
        for mode, kw in ((HG_AGG_RUNS, dict(group_col=0, ts_col=1, window_ms=10_000, value_col=2)), (HG_AGG_RUNS, dict(group_col=0, ts_col=-1, window_ms=0, value_col=2)),
                         (HG_AGG_HASH, dict(group_col=3, ts_col=1, window_ms=10_000, value_col=2))):
            exp = oracle.scan_aggregate(datas, schema.arrow_schema, 2, _to_oracle(preds), mode=mode, **kw)
            eng = Engine(device=0)
            got = eng.scan_aggregate(handle, _inputs(datas), preds, mode=mode, **kw)
            st = eng.stats()
            eng.close()
            assert st["path"] & 1 == 0 and got.num_rows == len(exp.count)
            assert got["count"].to_numpy().tolist() == exp.count.tolist()
            assert np.array_equal(got["sum"].to_numpy().view(np.uint64), exp.sum.view(np.uint64))
            assert np.array_equal(got["min"].to_numpy(), exp.min) and np.array_equal(got["max"].to_numpy(), exp.max)
            if kw["ts_col"] >= 0:
                assert got["bucket"].to_numpy().tolist() == exp.bucket.tolist()


def test_in_set_with_a_binary_predicate_and_on_an_append_table():
    """IN_SET next to a Binary predicate (three predicate kernels, one conjunction), and on the key of an Append-mode table: the same
    batches as the short IN list they stand for"""
    rng = np.random.default_rng(31)
    for append in (False, True):
        mode = UpdateMode.Append if append else UpdateMode.Overwrite
        user = pa.schema([pa.field("k", pa.uint32()), pa.field("ts", pa.int64()), pa.field("blob", pa.binary())] + ([] if append else [pa.field("v", pa.int16())]))
        schema = StorageSchema.try_new(user, 2, mode)
        handle = SchemaHandle(schema.arrow_schema, 2, mode)
        datas = []
        for f in range(3):
            n = 1500
            k = np.sort(rng.integers(0, 200, n))
            ts = T0 + rng.integers(0, 30, n)
            order = np.lexsort((ts, k))
            keep = np.ones(n, bool)
            keep[1:] = (k[order][1:] != k[order][:-1]) | (ts[order][1:] != ts[order][:-1])
            k, ts = k[order][keep], ts[order][keep]
            arrays = [pa.array(k, pa.uint32()), pa.array(ts, pa.int64()), pa.array([bytes([97 + int(x)]) * int(1 + x) for x in rng.integers(0, 6, len(k))], pa.binary())]
            if not append:
                arrays.append(pa.array(rng.integers(-5, 5, len(k)), pa.int16()))
            datas.append(sstgen.write_sst(schema, pa.RecordBatch.from_arrays(arrays, schema=user), seq=50 + f, cfg=WriteConfig(max_row_group_size=400), presorted=True))
        keys = rng.permutation(200)[:60].tolist()
        for rest in ([], [("blob", "ge", b"c")], [("blob", "in", [b"a", b"ccc"]), ("ts", "lt", T0 + 20)]):
            outs = []
            for op in ("in", "in_set"):
                eng = Engine(device=0)
                outs.append(list(eng.scan(handle, _inputs(datas), [("k", op, keys), *rest])))
                eng.close()
            assert sum(b.num_rows for b in outs[0]) > 0
            check_stream(outs[1], outs[0])


# ------------------------------------------------------------------------------------------------------------ codecs and encodings
@pytest.mark.parametrize("codec", [ParquetCompression.Snappy, ParquetCompression.Uncompressed, ParquetCompression.Zstd])
@pytest.mark.parametrize("kind", ["plain", "dict", "delta", "pages"])
def test_in_set_codecs_encodings_and_multi_page_chunks(codec, kind):
    rng = np.random.default_rng(41)
    schema = _schema()
    if kind == "dict":
        cfg = WriteConfig(compression=codec, max_row_group_size=2500, enable_dict=True)
    elif kind == "delta":
        cfg = WriteConfig(compression=codec, max_row_group_size=2500,
                          column_options={c: ColumnOptions(encoding=ParquetEncoding.DeltaBinaryPacked) for c in ("series_id", "ts", "tag")})
    else:
        cfg = WriteConfig(compression=codec, max_row_group_size=2500)
    if kind == "pages":
        cfg.write_bacth_size = 300                                   # several data pages per chunk
    datas = _overlapping(rng, schema, nfiles=2, cfgs=[cfg, cfg])
    if kind == "pages":
        md = pq.ParquetFile(io.BytesIO(datas[0])).metadata
        assert md.row_group(0).column(0).total_compressed_size > 0
    _check_scan(schema, datas, [("series_id", "in_set", rng.permutation(300)[:100].tolist()), ("tag", "in_set", list(range(0, 50, 2)))])


# ------------------------------------------------------------------------------------------------------------------------ pruning
def test_in_set_prunes_row_groups_by_the_sorted_set():
    """rows_decoded = the rows of exactly the row groups whose [min, max] holds a member of the set (pyarrow's reading of the
    statistics); without pruning every row is decoded and the result is the same; pruned row groups of a transient file never cross PCIe"""
    schema, datas, allcols = _big_files(40_000, 1_000_000, 6, rg=1000)
    rng = np.random.default_rng(61)
    values = np.concatenate([rng.choice(1_000_000, size=4, replace=False), np.arange(400_000, 430_000, 7)]).astype(np.uint64)
    sv = np.sort(values)
    want = 0
    for d in datas:
        md = pq.ParquetFile(io.BytesIO(d)).metadata
        for g in range(md.num_row_groups):
            s = md.row_group(g).column(0).statistics
            lo = np.searchsorted(sv, s.min, "left")
            if lo < len(sv) and sv[lo] <= s.max:
                want += md.row_group(g).num_rows
    preds = [("series_id", "in_set", values)]
    res = {}
    for flags in (0, HG_FLAG_NO_PRUNING):
        for resident in ((), (0, 1)):
            got, st = _scan(schema, datas, preds, flags=flags, resident=resident)
            res[flags, bool(resident)] = (pa.Table.from_batches(got), st)
            assert st["rows_decoded"] == (want if flags == 0 else st["rows_in_files"]), (flags, resident)
    assert 0 < want < 80_000 and res[0, False][1]["rows_in_files"] == 80_000
    base = res[0, False][0]
    assert base.num_rows == int(np.isin(allcols["series_id"], values).sum())
    for t, _ in res.values():
        assert t.equals(base)
    assert res[0, False][1]["bytes_h2d"] < res[HG_FLAG_NO_PRUNING, False][1]["bytes_h2d"] // 2


def test_in_set_adds_one_launch_and_other_calls_none():
    """one kernel for all the IN_SET predicates of a call, launched only when there is one"""
    schema, datas, _ = _big_files(20_000, 100_000, 7, tag_span=1 << 21)
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0, flags=HG_FLAG_NO_FUSED | HG_FLAG_NO_PRUNING)
    sst = _inputs(datas[:1])[0]
    eng.load_sst(handle, sst)
    ins = [SstInput(id=sst.id)]
    rng_pred = [("ts", "ge", T0)]
    kw = dict(group_col=0, ts_col=-1, window_ms=0, value_col=2)
    launches = []
    for preds in (rng_pred, rng_pred + [("series_id", "in_set", list(range(0, 100_000, 3)))],
                  rng_pred + [("series_id", "in_set", list(range(0, 100_000, 2))), ("tag", "in_set", np.arange(1 << 20))], [("series_id", "in_set", list(range(0, 100_000, 3)))],
                  [("series_id", "ge", 3)]):
        eng.scan_aggregate(handle, ins, preds, **kw)
        launches.append(eng.stats()["kernel_launches"])
    eng.close()
    assert launches[1] == launches[0] + 1 and launches[2] == launches[0] + 1, launches
    assert launches[3] == launches[0] == launches[4], launches                   # alone it takes the place of the comparison kernel


# ---------------------------------------------------------------------------------------------------------------------- refusals
def test_in_set_refusals():
    schema = _schema(extra=[pa.field("name", pa.binary())])
    cols = {"series_id": [1, 2], "ts": [T0, T0], "value": [1.0, 2.0], "tag": [1, 2], "name": [b"a", b"b"]}
    data = _write(schema, cols, 1)
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    for col in ("value", "name"):
        with pytest.raises(HgError) as ei:
            list(eng.scan(handle, _inputs([data]), [(col, "in_set", [1])]))
        assert ei.value.code == 2 and col in str(ei.value)
    L = lib()
    ins, keep = eng._descs(_inputs([data]))

    def raw_scan(op, count, ptr):
        p = (HgPredicate * 1)()
        p[0].column, p[0].op, p[0].in_count = 0, op, count
        p[0].in_values = ptr
        from horaedb_b200._ffi import ArrowArrayStream
        stream = ArrowArrayStream()
        return L.hg_scan_open(eng._h, C.byref(handle.desc), ins, C.c_size_t(1), p, C.c_size_t(1), None, C.c_size_t(0), 0, C.byref(stream))

    one = (C.c_uint64 * 1)(1)
    assert raw_scan(7, (1 << 24) + 1, one) == 1                 # more than HG_MAX_IN_SET values: refused before anything is read
    assert raw_scan(7, 1, None) == 1                            # null pointer
    assert raw_scan(8, 1, one) != 0                             # no such operator
    assert raw_scan(6, 65, one) == 1                            # IN keeps its limit
    with pytest.raises(HgError) as ei:
        eng.compact_to_sst(SchemaHandle(_schema().arrow_schema, 2), [], "/dev/null", shard_preds=[("series_id", "in_set", [1])])
    assert ei.value.code == 1
    assert list(eng.scan(handle, _inputs([data]), [("series_id", "in_set", [2])]))[0].num_rows == 1
    eng.close()
