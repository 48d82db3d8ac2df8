"""Predicates on Binary columns (`=`, `<>`, `<`, `<=`, `>`, `>=`, `IN`) on the GPU path: FilterExec in front of the merge (read.rs:459-480)
and PruningPredicate's min/max rewrite over the chunks' min_value / max_value.  Binary values order as arrow-rs BinaryArray: unsigned
bytes lexicographically, a proper prefix first; NULL fails every operator.

Model, independent of the library: pyarrow decodes every SST, `pyarrow.compute` filters each file's rows, the rows are merged in
(pk.., __seq__, stream) order, cut into batches like SortPreservingMergeExec, and oracle/merge_stream.py applies LastValueOperator or
BytesMergeOperator.  Rows, bytes, validity and batch boundaries must be identical."""
import io

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import (HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_FUSED, HG_FLAG_NO_PRUNING, Engine, SchemaHandle, SstInput)
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode
from oracle.merge_stream import BytesMergeOperator, LastValueOperator, MergeStream

from helpers import arrays_equal, arrow_schema, record_batch
from test_gpu_binary_append import _check
from test_gpu_binary_encodings import USER, _encodings, _write_direct, pages

pytestmark = pytest.mark.gpu
_ids = iter(range(130_000_000, 134_000_000))
CODECS = [ParquetCompression.Snappy, ParquetCompression.Uncompressed, ParquetCompression.Zstd]
OPS = {"eq": pc.equal, "ne": pc.not_equal, "lt": pc.less, "le": pc.less_equal, "gt": pc.greater, "ge": pc.greater_equal}

# stored values around the literals: prefixes of each other, 8- and 16-byte shared prefixes differing after them in both directions,
# bytes 0x00 / 0xff, a value longer than 64 KiB and its 64 KiB prefix
P8, P16 = b"prefix08", b"prefix16prefix16"
BIG = b"L" * 70_000
POOL = [b"", b"\x00", b"\x00\x00", b"\x01", b"\x7f", b"\x80", b"\xff", b"\xff" * 8, b"\xff" * 9, b"\xff" * 10, b"ab", b"ab\x00", b"abc",
        b"abcd", b"abd", P8, P8 + b"\x00", P8 + b"A", P8 + b"M", P8 + b"Z", P8[:7] + b"\x00", P8[:7] + b"\xff" + b"tail", P16, P16 + b"\x00",
        P16 + b"M", P16[:15] + b"\x00", P16[:15] + b"\xff", P16 + b"Mzz" * 5, b"L" * 65_536, BIG]
LITERALS = [b"", b"\x00", b"\xff" * 9, b"ab", P8, b"abcd", P8 + b"A\x00", P8 + b"M", P16 + b"M", P16[:15] + b"\x80", b"L" * 65_536, b"zzz"]


# ------------------------------------------------------------------------------------------------------------------- model
def _mask(t, preds):
    m = pa.array(np.ones(t.num_rows, bool))
    for col, op, lit in preds:
        a = t[col]
        if op == "in":
            x = pc.is_in(a, value_set=pa.array(list(lit), a.type))
        else:
            x = OPS[op](a, pa.scalar(lit, a.type))
        m = pc.and_(m, pc.fill_null(x, False))
    return m


def _as_batch(t):
    t = t.combine_chunks()
    return t.to_batches()[0] if t.num_rows else None


def model_scan(schema: StorageSchema, datas, preds, append: bool, keep_builtin: bool, batch_size=8192):
    live = [d for d in datas if pq.read_metadata(io.BytesIO(d)).num_rows]
    if not live:
        return []
    tables = [pq.read_table(io.BytesIO(d)) for d in live]
    names = schema.arrow_schema.names
    if len(tables) == 1:
        # ParquetExec's batches (<= batch_size rows, never across a row group), each filtered by FilterExec
        md = pq.ParquetFile(io.BytesIO(live[0])).metadata
        batches, row = [], 0
        for g in range(md.num_row_groups):
            n = md.row_group(g).num_rows
            for lo in range(0, n, batch_size):
                s = tables[0].slice(row + lo, min(batch_size, n - lo))
                batches.append(_as_batch(s.filter(_mask(s, preds))))
            row += n
        batches = [b for b in batches if b is not None]
    else:
        tables = [t.filter(_mask(t, preds)) for t in tables]
        allrows = pa.concat_tables(tables).combine_chunks()
        src = np.concatenate([np.full(t.num_rows, i) for i, t in enumerate(tables)])
        pos = np.concatenate([np.arange(t.num_rows) for t in tables])
        keys = [pos, src, allrows["__seq__"].to_numpy()] + [allrows[names[k]].to_numpy() for k in reversed(range(schema.num_primary_keys))]
        merged = allrows.take(pa.array(np.lexsort(keys)))
        batches = [_as_batch(merged.slice(lo, batch_size)) for lo in range(0, merged.num_rows, batch_size)]
    op = BytesMergeOperator(schema.value_idxes) if append else LastValueOperator()
    return list(MergeStream(batches, schema.num_primary_keys, op, keep_builtin))


def _project(batches, cols):
    return [pa.RecordBatch.from_arrays([b.column(c) for c in cols], names=[b.schema.names[c] for c in cols]) for b in batches]


# -------------------------------------------------------------------------------------------------------------------- data
def _rows(rng, n, keyspace, f, null_rate=0.1, big=True, append=False):
    """Sorted unique (pk1, pk2); blob from POOL and random bytes, idx short labels; a key is NULL in at most one file.  `append`: no empty
    values, so that no run of several rows concatenates to zero bytes (which BytesMergeOperator cannot assemble, operator.rs:80-92)."""
    pk1 = np.sort(rng.integers(0, keyspace, n))
    pk2 = rng.integers(-3, 4, n)
    order = np.lexsort((pk2, pk1))
    pk1, pk2 = pk1[order], pk2[order]
    keep = np.ones(len(pk1), bool)
    keep[1:] = (pk1[1:] != pk1[:-1]) | (pk2[1:] != pk2[:-1])
    pk1, pk2 = pk1[keep], pk2[keep]
    blob = []
    for i in range(len(pk1)):
        r = rng.random()
        if (int(pk1[i]) + f) % 7 == 0 and r < null_rate * 7:
            blob.append(None)
        elif r < 0.7:
            v = POOL[int(rng.integers(0, len(POOL)))]
            blob.append(v if big or len(v) < 1000 else v[:20])
        else:
            blob.append(rng.bytes(int(rng.integers(0, 24))))
    if append:
        blob = [b"\x00" if v == b"" else v for v in blob]
    idx = [[b"label-a", b"label-b", b"label-" if append else b"", b"label-aa"][int(rng.integers(0, 4))] for _ in range(len(pk1))]
    return record_batch(USER, {"pk1": pk1.tolist(), "pk2": pk2.tolist(), "blob": blob, "idx": idx})


def _enc_cfg(codec, kind, rg=600):
    if kind == "plain":
        return WriteConfig(compression=codec, max_row_group_size=rg)
    if kind == "dict":
        return WriteConfig(compression=codec, max_row_group_size=rg, enable_dict=True)
    enc = ParquetEncoding.DeltaLengthByteArray if kind == "dlba" else ParquetEncoding.DeltaByteArray
    return WriteConfig(compression=codec, max_row_group_size=rg, column_options={c: ColumnOptions(encoding=enc) for c in ("blob", "idx")})


def _mixed_files(schema, rng, append, codec=ParquetCompression.Snappy, n=1200):
    """one file per Binary encoding (PLAIN, DELTA_LENGTH_BYTE_ARRAY, dictionary, DELTA_BYTE_ARRAY), overlapping keys"""
    out = []
    for f, kind in enumerate(("plain", "dlba", "dict", "dba")):
        out.append(sstgen.write_sst(schema, _rows(rng, n, 900, f, append=append), seq=10 + f, cfg=_enc_cfg(codec, kind), presorted=True))
    return out


class Runner:
    def __init__(self, append, datas):
        self.append = append
        self.mode = UpdateMode.Append if append else UpdateMode.Overwrite
        self.schema = StorageSchema.try_new(USER, 2, self.mode)
        self.handle = SchemaHandle(self.schema.arrow_schema, 2, self.mode)
        self.datas = datas
        self.eng = Engine(device=0)
        self.ids = [next(_ids) for _ in datas]
        for i, d in zip(self.ids, datas):
            self.eng.load_sst(self.handle, SstInput(id=i, data=d))

    def inputs(self, how):
        if how == "resident":
            return [SstInput(id=i) for i in self.ids]
        if how == "transient":
            return [SstInput(id=next(_ids), data=d) for d in self.datas]
        return [SstInput(id=i) if k % 2 else SstInput(id=next(_ids), data=d) for k, (i, d) in enumerate(zip(self.ids, self.datas))]   # mixed

    def check(self, preds, how="resident", keep_builtin=False, projection=None, flags=0):
        self.eng.set_flags(flags)
        got = list(self.eng.scan(self.handle, self.inputs(how), preds, projection, keep_builtin))
        self.eng.set_flags(0)
        exp = model_scan(self.schema, self.datas, preds, self.append, keep_builtin)
        if projection is not None:
            exp = _project(exp, projection)
        try:
            _check(got, exp)
        except AssertionError as ex:
            raise AssertionError(f"preds={[(c, o, l if not isinstance(l, bytes) or len(l) < 40 else l[:20] + b'..') for c, o, l in preds]} "
                                 f"how={how} keep_builtin={keep_builtin} projection={projection} flags={flags}: {ex}") from None
        return sum(b.num_rows for b in got)

    def close(self):
        self.eng.close()


# ------------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("append", [False, True])
def test_every_operator_and_edge_literal(append):
    rng = np.random.default_rng(101)
    r = Runner(append, _mixed_files(StorageSchema.try_new(USER, 2, UpdateMode.Append if append else UpdateMode.Overwrite), rng, append))
    total = 0
    for lit in LITERALS:
        for op in OPS:
            total += r.check([("blob", op, lit)])
    assert total > 0
    # the same calls on transient and mixed loads, without pruning, with the builtin columns and with the column projected away
    for lit in (b"", P8, P16 + b"M", b"L" * 65_536):
        for op in ("eq", "lt", "ge", "ne"):
            r.check([("blob", op, lit)], how="transient")
            r.check([("blob", op, lit)], how="mixed", keep_builtin=True)
            r.check([("blob", op, lit)], flags=HG_FLAG_NO_PRUNING)
            r.check([("blob", op, lit)], projection=[0, 3])
    r.close()


@pytest.mark.parametrize("append", [False, True])
def test_in_lists_and_conjunctions(append):
    rng = np.random.default_rng(103)
    r = Runner(append, _mixed_files(StorageSchema.try_new(USER, 2, UpdateMode.Append if append else UpdateMode.Overwrite), rng, append))
    in1 = [P8 + b"M"]
    in8 = [b"", b"ab", b"ab", P16, b"\xff" * 9, b"nothere", P8 + b"Z", b"L" * 65_536]
    in64 = [POOL[int(i)] for i in rng.integers(0, len(POOL), 40)] + [rng.bytes(int(rng.integers(0, 12))) for _ in range(24)]
    cases = [[("blob", "in", in1)], [("blob", "in", in8)], [("blob", "in", in64)], [("blob", "in", [])],
             [("blob", "eq", b"ab"), ("blob", "eq", b"abc")],                                    # contradictory
             [("blob", "ge", P8), ("blob", "lt", P8 + b"N")],                                    # a prefix range
             [("blob", "gt", b"ab"), ("pk2", "ge", 0)], [("pk2", "lt", 2), ("blob", "in", in8), ("pk1", "gt", 100)],
             [("blob", "ne", b""), ("idx", "eq", b"label-a")], [("idx", "in", [b"", b"label-aa"]), ("blob", "le", P16)],
             [("idx", "lt", b"label-b"), ("idx", "ge", b"label-a"), ("blob", "ne", P8)]]
    for preds in cases:
        for how in ("resident", "transient", "mixed"):
            r.check(preds, how=how)
        r.check(preds, keep_builtin=True, flags=HG_FLAG_NO_PRUNING)
        r.check(preds, projection=[1, 0])
    r.close()


@pytest.mark.parametrize("codec", CODECS)
def test_pages_codecs_and_encodings(codec):
    """V1 and V2 pages, several pages per chunk, every Binary encoding, each codec; Overwrite and Append."""
    rng = np.random.default_rng(107)
    for append in (False, True):
        schema = StorageSchema.try_new(USER, 2, UpdateMode.Append if append else UpdateMode.Overwrite)
        batches = [_rows(rng, 1500, 1200, f, big=False, append=append) for f in range(4)]
        datas = [_write_direct(schema, b, 200 + i, codec, ver, 600, enc)
                 for i, (b, ver, enc) in enumerate(zip(batches, ("1.0", "2.0", "2.0", "1.0"), ("PLAIN", "DELTA_LENGTH_BYTE_ARRAY", "DELTA_BYTE_ARRAY", "DELTA_BYTE_ARRAY")))]
        assert len(pages(datas[1], 0, 2)) > 1 and "DELTA_BYTE_ARRAY" in _encodings(datas[2])
        r = Runner(append, datas)
        for preds in ([("blob", "ge", P8), ("blob", "lt", P8 + b"\xff")], [("blob", "in", [b"ab", b"", P16 + b"M"])], [("blob", "gt", b"\x7f")],
                      [("idx", "eq", b"label-b")]):
            r.check(preds)
            r.check(preds, how="transient")
        r.close()


def test_dictionary_fallback_mid_chunk_and_null_heavy_chunks():
    """A dictionary chunk that falls back to PLAIN pages mid-chunk; chunks almost all NULL and row groups whose Binary chunk is all NULL
    (PruningPredicate drops them: NULL fails every operator, `<>` included)."""
    rng = np.random.default_rng(109)
    n = 8192
    for append in (False, True):
        schema = StorageSchema.try_new(USER, 2, UpdateMode.Append if append else UpdateMode.Overwrite)
        pk1 = np.arange(n, dtype=np.uint64) * 2
        blob = [None if k % 11 == 0 else (P16 + rng.bytes(184)) for k in range(n)]
        fb = sstgen.write_sst(schema, record_batch(USER, {"pk1": pk1.tolist(), "pk2": [1] * n, "blob": blob, "idx": [b"ab"] * n}), seq=10,
                              cfg=WriteConfig(enable_dict=True), presorted=True)
        assert {(t, e) for t, e, _, _, _ in pages(fb, 0, 2)} >= {(0, 8), (0, 0)}
        m = 3000
        pk1 = np.arange(m, dtype=np.uint64) * 5 + 1
        nul = [None if (i // 500) % 2 == 0 or rng.random() < 0.9 else POOL[int(rng.integers(0, 20))] for i in range(m)]
        fn = sstgen.write_sst(schema, record_batch(USER, {"pk1": pk1.tolist(), "pk2": [0] * m, "blob": nul, "idx": [None] * m}), seq=11,
                              cfg=WriteConfig(max_row_group_size=500), presorted=True)
        md = pq.ParquetFile(io.BytesIO(fn)).metadata
        assert md.row_group(0).column(2).statistics.null_count == 500
        lit = sorted(v for v in nul if v is not None)[0]
        for datas in ([fb], [fn], [fb, fn]):
            r = Runner(append, datas)
            for preds in ([("blob", "ne", b"x")], [("blob", "ge", P16)], [("blob", "eq", lit)], [("idx", "ne", b"")], [("blob", "in", [lit, b""])]):
                r.check(preds)
                r.check(preds, how="transient")
            r.eng.scan(r.handle, r.inputs("resident"), [("blob", "ne", b"x")]).read_all()
            if datas == [fn]:
                st = r.eng.stats()                    # the all-NULL row groups are pruned, `<>` prunes nothing else
                assert st["rows_decoded"] == sum(md.row_group(g).num_rows for g in range(md.num_row_groups)
                                                 if md.row_group(g).column(2).statistics.null_count < md.row_group(g).num_rows)
            r.close()


def test_pruning_by_binary_statistics():
    """Files whose Binary column is sorted within each file: rows_decoded for `b = x` is the rows of the row groups whose
    [min_value, max_value] can hold x; `<>` and HG_FLAG_NO_PRUNING decode everything."""
    rng = np.random.default_rng(113)
    schema = StorageSchema.try_new(USER, 2)
    datas = []
    for f in range(3):
        n = 2000
        vals = sorted([POOL[int(i)] for i in rng.integers(0, 27, n - 40)] + [rng.bytes(int(rng.integers(0, 12))) for _ in range(40)])
        pk1 = np.arange(n, dtype=np.uint64) * 3 + f
        datas.append(sstgen.write_sst(schema, record_batch(USER, {"pk1": pk1.tolist(), "pk2": [0] * n, "blob": vals, "idx": [b"i"] * n}), seq=20 + f,
                                      cfg=WriteConfig(max_row_group_size=250, compression=ParquetCompression.Uncompressed), presorted=True))
    r = Runner(False, datas)
    mds = [pq.ParquetFile(io.BytesIO(d)).metadata for d in datas]

    def can_hold(x, op):
        rows = 0
        for md in mds:
            for g in range(md.num_row_groups):
                s = md.row_group(g).column(2).statistics
                mn, mx = s.min, s.max
                ok = {"eq": mn <= x <= mx, "lt": mn < x, "le": mn <= x, "gt": mx > x, "ge": mx >= x, "ne": True}[op]
                rows += md.row_group(g).num_rows if ok else 0
        return rows

    total = sum(md.num_rows for md in mds)
    for x in [b"", b"\x00", b"ab", b"abc", P8 + b"M", P16, b"\xff" * 9, b"zzz"]:
        for op in ("eq", "lt", "ge", "ne"):
            r.check([("blob", op, x)])
            assert r.eng.stats()["rows_decoded"] == can_hold(x, op), (x, op)
            r.check([("blob", op, x)], flags=HG_FLAG_NO_PRUNING)
            assert r.eng.stats()["rows_decoded"] == total
    r.check([("blob", "eq", P8 + b"M")])
    assert 0 < r.eng.stats()["rows_decoded"] < total // 3
    r.close()


def test_launches_with_and_without_binary_predicates():
    """A Binary predicate adds exactly one kernel (eval_binary_predicates) next to fixed-width ones, and replaces eval_predicates when
    the conjunction has no fixed-width predicate."""
    rng = np.random.default_rng(127)
    schema = StorageSchema.try_new(USER, 2)
    r = Runner(False, [sstgen.write_sst(schema, _rows(rng, 3000, 100_000, 0, big=False), seq=5, cfg=_enc_cfg(ParquetCompression.Snappy, "plain"),
                                        presorted=True)])
    launches = []
    for preds in ([("pk2", "ge", -100)], [("pk2", "ge", -100), ("blob", "ne", b"\x01zz")], [("blob", "ne", b"\x01zz")]):
        r.check(preds)
        launches.append(r.eng.stats()["kernel_launches"])
    assert launches[1] == launches[0] + 1 and launches[2] == launches[0], launches
    r.close()


# --------------------------------------------------------------------------------------------------------------- aggregates
GUSER = arrow_schema([("pk1", "uint64"), ("ts", "int64"), ("v", "float64"), ("tag", "uint32"), ("b", "binary")])


def _agg_model(datas, schema, preds, group, ts, w, value):
    rows = pa.Table.from_batches(model_scan(schema, datas, preds, False, False), schema=schema.user_schema()) if datas else None
    groups = {}
    order = []
    for pk1, t, v, tag in zip(*(rows[c].to_pylist() for c in ("pk1", "ts", "v", "tag"))):
        key = ({"pk1": pk1, "tag": tag}[group], t // w * w)                    # (ts >= 0 here: truncation = floor)
        if key not in groups:
            groups[key] = [0, 0.0, None, None]
            order.append(key)
        g = groups[key]
        g[0] += 1
        if v is not None:
            g[1] += v
            g[2] = v if g[2] is None or v < g[2] else g[2]
            g[3] = v if g[3] is None or v > g[3] else g[3]
    return [(k[0], k[1], g[0], g[1], g[2], g[3]) for k, g in ((k, groups[k]) for k in sorted(order))]


@pytest.mark.parametrize("how", ["resident", "transient"])
def test_aggregates_with_binary_predicates(how):
    """hg_scan_aggregate / _device on Overwrite tables with the Binary column only in the predicate, RUNS and HASH mode: the fused kernel
    declines every such call (path 0), the general pipeline filters before the merge; f64 sums bit for bit."""
    rng = np.random.default_rng(131)
    schema = StorageSchema.try_new(GUSER, 2)
    handle = SchemaHandle(schema.arrow_schema, 2)
    datas = []
    for f in range(3):
        n = 1500
        pk1 = np.sort(rng.integers(0, 40, n)).astype(np.uint64)
        ts = np.arange(n, dtype=np.int64) * 1000 + f * 137
        v = rng.normal(size=n).round(3)
        tag = rng.integers(0, 5, n).astype(np.uint32)
        b = [POOL[int(i)] if i < 27 else None for i in rng.integers(0, 30, n)]
        datas.append(sstgen.write_sst(schema, record_batch(GUSER, {"pk1": pk1.tolist(), "ts": ts.tolist(), "v": v.tolist(), "tag": tag.tolist(), "b": b}),
                                      seq=30 + f, cfg=WriteConfig(max_row_group_size=500, compression=ParquetCompression.Uncompressed)))
    eng = Engine(device=0)
    ids = [next(_ids) for _ in datas]
    for i, d in zip(ids, datas):
        eng.load_sst(handle, SstInput(id=i, data=d))
    ins = (lambda: [SstInput(id=i) for i in ids]) if how == "resident" else (lambda: [SstInput(id=next(_ids), data=d) for d in datas])
    for preds in ([("b", "eq", P8 + b"M")], [("b", "ge", b"ab"), ("ts", "lt", 900_000)], [("b", "in", [b"", b"\xff" * 9, P16])], [("b", "ne", b"abc")],
                  [("pk1", "ge", 3), ("b", "lt", P8)]):
        for group, mode in (("pk1", HG_AGG_RUNS), ("pk1", HG_AGG_HASH), ("tag", HG_AGG_HASH)):
            kw = dict(group_col=GUSER.names.index(group), ts_col=1, window_ms=60_000, value_col=2, mode=mode)
            exp = _agg_model(datas, schema, preds, group, 1, 60_000, "v")
            for flags in (0, HG_FLAG_NO_FUSED, HG_FLAG_NO_PRUNING):
                eng.set_flags(flags)
                got = eng.scan_aggregate(handle, ins(), preds, **kw)
                assert eng.stats()["path"] & 1 == 0
                rows = list(zip(got.column(0).to_pylist(), got["bucket"].to_pylist(), got["count"].to_pylist(), got["sum"].to_pylist(),
                                got["min"].to_pylist(), got["max"].to_pylist()))
                assert len(rows) == len(exp) > 0, (preds, group, mode, flags)
                for a, e in zip(rows, exp):
                    assert a[:3] == e[:3] and np.float64(a[3]).tobytes() == np.float64(e[3]).tobytes() and a[4:] == e[4:], (preds, group, a, e)
                dev = eng.scan_aggregate_device(handle, ins(), preds, **kw)
                assert dev.num_groups == len(exp) and eng.stats()["path"] & 1 == 0
            eng.set_flags(0)
    eng.close()
