"""Host only: split-block bloom filters on the read side and in the Python mirror, without a GPU.

* tests/bloom_model.py (xxHash64 + SBBF from the spec, with a footer walk of its own) reproduces pyarrow's bitsets bit for bit, for
  every primitive type, NaN, signed zeros and nulls;
* hg_parquet_bloom_info / hg_parquet_bloom_probe read pyarrow's filters as the model does, and ignore damaged ones;
* hg_plan_row_groups prunes by them after statistics, for `=` / `IN` only, and never with a literal the column cannot represent;
* config.resolve_bloom_filters and what ObjectBasedStorage sends to the GPU writer."""
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import bloom_model as M
from horaedb_b200 import _ffi, sstgen
from horaedb_b200.config import ColumnOptions, StorageConfig, WriteConfig, resolve_bloom_filters, resolve_column_options
from horaedb_b200.types import StorageSchema

from helpers import arrow_schema, record_batch

TYPES = [pa.uint8(), pa.int8(), pa.uint16(), pa.int16(), pa.uint32(), pa.int32(), pa.uint64(), pa.int64(), pa.float32(), pa.float64()]
BLOOM = {"ndv": 1_000_000, "fpp": 0.05}


def _column(t, n, rng, null_rate=0.1):
    if pa.types.is_floating(t):
        v = rng.standard_normal(n).astype(t.to_pandas_dtype())
        v[:6] = [np.nan, -0.0, 0.0, np.inf, -np.inf, np.float64(np.nan) * -1]
        v[6] = np.array([0x7ff8000000000123], dtype=np.uint64).view(np.float64)[0] if t == pa.float64() else \
            np.array([0x7fc00123], dtype=np.uint32).view(np.float32)[0]            # a NaN with a payload
    else:
        info = np.iinfo(t.to_pandas_dtype())
        v = rng.integers(info.min, info.max, n, dtype=t.to_pandas_dtype(), endpoint=True)
    return pa.array(v, t, mask=rng.random(n) < null_rate)


def _typed_file(rg_rows=700, n=2000, seed=3):
    rng = np.random.default_rng(seed)
    cols = {f"c{i}": _column(t, n, rng) for i, t in enumerate(TYPES)}
    cols["allnull"] = pa.array([None] * n, pa.int64())
    tbl = pa.table(cols)
    sink = io.BytesIO()
    pq.write_table(tbl, sink, row_group_size=rg_rows, bloom_filter_options={c: BLOOM for c in cols})
    return tbl, sink.getvalue()


@pytest.fixture(scope="module")
def typed_file():
    return _typed_file()


def test_xxh64_anchors():
    assert M.xxh64(b"", 0) == 0xEF46DB3751D8E999
    x4 = np.array([0, 1, 0xdeadbeef, 0xffffffff], dtype=np.uint32)
    x8 = np.array([0, 1, 0x0123456789abcdef, 2**64 - 1], dtype=np.uint64)
    assert [int(h) for h in M.hash_phys(x4)] == [M.xxh64(int(v).to_bytes(4, "little")) for v in x4]
    assert [int(h) for h in M.hash_phys(x8)] == [M.xxh64(int(v).to_bytes(8, "little")) for v in x8]
    for n in (3, 17, 40, 77):                      # the long-input path of the scalar form (stripes of 32 bytes)
        assert M.xxh64(bytes(range(n))) != M.xxh64(bytes(range(1, n + 1)))


def test_model_reproduces_pyarrow_bitsets(typed_file):
    tbl, data = typed_file
    blooms = M.footer_blooms(data)
    assert len(blooms) == 3 * tbl.num_columns
    for (g, c), ent in blooms.items():
        nbytes, hlen, bits = M.read_filter(data, ent["offset"])
        assert nbytes == 1 << 20 and ent["length"] == hlen + nbytes
        rows = tbl.column(c).slice(g * 700, 700)
        assert bits == M.build(M.phys_values(rows), nbytes), (g, tbl.column_names[c])
    # the all-null chunk's filter is empty
    assert not any(M.read_filter(data, blooms[(0, tbl.num_columns - 1)]["offset"])[2])


def test_library_reads_pyarrow_filters_like_the_model(typed_file):
    tbl, data = typed_file
    rng = np.random.default_rng(9)
    blooms = M.footer_blooms(data)
    for (g, c), ent in blooms.items():
        info = _ffi.parquet_bloom_info(data, g, c)
        nbytes, hlen, bits = M.read_filter(data, ent["offset"])
        assert info == {"offset": ent["offset"], "length": ent["length"], "num_bytes": nbytes, "bitset_offset": ent["offset"] + hlen, "usable": 1}
        t = tbl.schema.field(c).type
        present = M.phys_values(tbl.column(c).slice(g * 700, 700))[:40]
        width = 8 if t in (pa.uint64(), pa.int64(), pa.float64()) else 4
        others = rng.integers(0, 2**63, 200, dtype=np.uint64).astype(np.uint32 if width == 4 else np.uint64)
        for v in list(present) + list(others):
            h = int(M.hash_phys(np.array([v], dtype=np.uint32 if width == 4 else np.uint64))[0])
            got = _ffi.parquet_bloom_probe(data, g, c, int(v).to_bytes(width, "little"))
            assert got == M.may_contain(bits, h)
        assert all(_ffi.parquet_bloom_probe(data, g, c, int(v).to_bytes(width, "little")) for v in present)


def test_chunks_without_filters_and_binary_chunks():
    tbl = pa.table({"a": pa.array([1, 2, 3], pa.int64()), "b": pa.array([b"x", b"y", b"z"], pa.binary())})
    sink = io.BytesIO()
    pq.write_table(tbl, sink, bloom_filter_options={"b": BLOOM})
    data = sink.getvalue()
    assert _ffi.parquet_bloom_info(data, 0, 0) == {"offset": -1, "length": -1, "num_bytes": 0, "bitset_offset": 0, "usable": 0}
    b = _ffi.parquet_bloom_info(data, 0, 1)
    assert b["offset"] > 0 and b["usable"] == 0              # binary chunks keep no filter
    assert _ffi.parquet_bloom_probe(data, 0, 0, (7).to_bytes(8, "little"))
    with pytest.raises(_ffi.HgError):
        _ffi.parquet_bloom_probe(data, 0, 0, b"\0\0")


PLAN_SCHEMA = arrow_schema([("k", "uint64"), ("ts", "int64"), ("u8", "uint8"), ("i16", "int16"), ("f32", "float32"), ("f64", "float64"),
                            ("rid", "uint64")])


def _plan_file(bloom_cols, rg_rows=500, n=4000, seed=11):
    rng = np.random.default_rng(seed)
    st = StorageSchema.try_new(PLAN_SCHEMA, 2)
    f64 = rng.standard_normal(n).round(2)
    f64[10], f64[20], f64[30] = -0.0, np.nan, 0.5
    cols = {"k": np.sort(rng.integers(0, 50, n)).tolist(), "ts": rng.integers(0, 10**6, n).tolist(),
            "u8": rng.integers(0, 200, n).tolist(), "i16": rng.integers(-300, 300, n).tolist(),
            "f32": f64.astype(np.float32).tolist(), "f64": f64.tolist(),
            "rid": rng.permutation(np.arange(1, n + 1, dtype=np.uint64) * 1_000_003).tolist()}
    batch = record_batch(PLAN_SCHEMA, cols)
    cfg = WriteConfig(max_row_group_size=rg_rows, column_options={c: ColumnOptions(enable_bloom_filter=True) for c in bloom_cols})
    return st, batch, sstgen.write_sst(st, batch, 1, cfg)


def _patch_varint(data: bytearray, at, value):
    """Overwrites the zigzag varint at [a, b) with `value`, padded to the same length (an over-long varint is still a varint)."""
    a, b = at
    z = (value << 1) ^ (value >> 63)
    assert z < 1 << (7 * (b - a))
    for i in range(a, b):
        data[i] = (z & 0x7f) | (0x80 if i + 1 < b else 0)
        z >>= 7


def test_damaged_filters_are_ignored():
    st, batch, good = _plan_file(["rid"])
    schema = _ffi.SchemaHandle(st.arrow_schema, 2)
    blooms = M.footer_blooms(good)
    ent = blooms[(1, 6)]
    off = ent["offset"]
    nb_at = (off + 1, off + 5)                                # numBytes varint (1 MiB: 4 bytes)
    damages = {
        "numBytes not a power of two": lambda d: _patch_varint(d, nb_at, (1 << 20) + 32),
        "numBytes beyond the length": lambda d: _patch_varint(d, nb_at, 1 << 21),
        "numBytes below 32": lambda d: _patch_varint(d, nb_at, 16),
        "unknown algorithm": lambda d: d.__setitem__(off + 6, 0x2c),
        "unknown hash": lambda d: d.__setitem__(off + 10, 0x2c),
        "unknown compression": lambda d: d.__setitem__(off + 14, 0x2c),
        "offset before the data": lambda d: _patch_varint(d, ent["offset_at"], 2),
        "offset past the end": lambda d: _patch_varint(d, ent["offset_at"], len(good) + 100),
        "offset into a page": lambda d: _patch_varint(d, ent["offset_at"], 4),
        "length too short": lambda d: _patch_varint(d, ent["length_at"], 100),
        "negative length": lambda d: _patch_varint(d, ent["length_at"], -5),
    }
    assert good[off + 6] == 0x1c and good[off + 10] == 0x1c and good[off + 14] == 0x1c
    absent = [("rid", "eq", 2_000_006_001)]                             # inside every row group's min / max, in no filter
    assert _ffi.plan_row_groups(schema, good, absent) == [0] * 8
    _, _, without = _plan_file([])
    assert _ffi.plan_row_groups(schema, without, absent) == [1] * 8     # statistics alone keep every row group
    for why, damage in damages.items():
        d = bytearray(good)
        damage(d)
        d = bytes(d)
        assert _ffi.parquet_bloom_info(d, 1, 6)["usable"] == 0, why
        assert _ffi.parquet_bloom_info(d, 2, 6)["usable"] == 1, why
        assert _ffi.parquet_bloom_probe(d, 1, 6, (2_000_006_001).to_bytes(8, "little")), why
        # the planner falls back to statistics for that chunk only
        assert _ffi.plan_row_groups(schema, d, absent) == [0, 1, 0, 0, 0, 0, 0, 0], why


# ---------------------------------------------------------------------------------------------------------- the planner
def _model_keep(data, st, preds, stats_keep):
    tbl = pq.read_table(io.BytesIO(data))
    blooms = M.footer_blooms(data)
    out = []
    for g, k in enumerate(stats_keep):
        for col, op, lit in preds:
            c = tbl.column_names.index(col)
            ent = blooms.get((g, c), {"offset": -1})
            if k and ent["offset"] >= 0 and not M.bloom_keeps(M.read_filter(data, ent["offset"])[2], st.arrow_schema.field(c).type, op, lit):
                k = 0
        out.append(k)
    return out


PREDS = [
    [("rid", "eq", 1_000_003 * 17)],                                     # present in one row group
    [("rid", "eq", 2_000_006_001)],                                          # absent everywhere (inside every row group's min / max)
    [("rid", "in", [1_000_003 * 5, 1_000_003 * 3999, 2_000_006_001])],
    [("rid", "in", [2_000_006_001, 2_000_007, 3_000_010])],
    [("rid", "eq", 2_000_006_001), ("u8", "eq", 3)],
    [("i16", "eq", -7), ("rid", "ne", 2_000_006_001)],                             # NE never uses a filter
    [("f64", "eq", -0.0)], [("f64", "eq", 0.0)], [("f64", "eq", float("nan"))], [("f64", "eq", 0.5)],
    [("f64", "in", [-0.0, 0.25])],
    [("f32", "eq", 0.5)], [("f32", "eq", 0.1)],                          # 0.1 is no f32: never probed
    [("f32", "in", [0.5, 0.1])], [("f32", "eq", float("nan"))],
    [("rid", "lt", 999), ("rid", "ge", 5)],
]


@pytest.mark.parametrize("pi", range(len(PREDS)))
def test_planner_prunes_by_filters_after_statistics(pi):
    preds = PREDS[pi]
    st, _, with_f = _plan_file(["rid", "u8", "i16", "f32", "f64"])
    _, _, without = _plan_file([])
    schema = _ffi.SchemaHandle(st.arrow_schema, 2)
    stats_keep = _ffi.plan_row_groups(schema, without, preds)
    got = _ffi.plan_row_groups(schema, with_f, preds)
    assert got == _model_keep(with_f, st, preds, stats_keep)
    assert all(a <= b for a, b in zip(got, stats_keep))
    # never drops a row group that holds a matching row
    tbl = pq.read_table(io.BytesIO(with_f))
    for g in range(len(got)):
        rows = tbl.slice(g * 500, 500)
        m = np.ones(rows.num_rows, dtype=bool)
        for col, op, lit in preds:
            v = rows[col].to_numpy(zero_copy_only=False)
            if op == "eq":
                m &= (v.view(np.uint64) == np.array([lit], np.float64).view(np.uint64)[0]) if col == "f64" else (v == lit)
            elif op == "in":
                m &= np.isin(v, lit)
            elif op == "ne":
                m &= v != lit
            elif op == "lt":
                m &= v < lit
            elif op == "ge":
                m &= v >= lit
        if m.any() and stats_keep[g]:
            assert got[g] == 1, (g, preds)


def test_literals_outside_the_column_type_are_refused_before_any_pruning():
    st, _, data = _plan_file(["u8"])
    with pytest.raises(_ffi.HgError):
        _ffi.plan_row_groups(_ffi.SchemaHandle(st.arrow_schema, 2), data, [("u8", "eq", 300)])


def test_planner_prunes_point_lookups():
    st, batch, data = _plan_file(["rid"])
    schema = _ffi.SchemaHandle(st.arrow_schema, 2)
    rid = batch.column(6).to_numpy()
    keep = _ffi.plan_row_groups(schema, data, [("rid", "eq", int(rid[1234]))])
    assert keep[1234 // 500] == 1 and sum(keep) <= 2          # statistics alone keep every row group (rid is not sorted)
    _, _, without = _plan_file([])
    assert sum(_ffi.plan_row_groups(schema, without, [("rid", "eq", int(rid[1234]))])) == len(keep)


# ---------------------------------------------------------------------------------------------------------- the Python mirror
USER = arrow_schema([("k", "uint64"), ("ts", "int64"), ("v", "float64"), ("t", "uint16")])
SCHEMA = StorageSchema.try_new(USER, 2).arrow_schema


def test_resolve_bloom_filters():
    assert resolve_bloom_filters(WriteConfig(), SCHEMA) is None
    assert resolve_bloom_filters(WriteConfig(enable_bloom_filter=True), SCHEMA) == [True] * 6
    cfg = WriteConfig(enable_bloom_filter=True, column_options={"ts": ColumnOptions(enable_bloom_filter=False), "nope": ColumnOptions(enable_bloom_filter=False)})
    assert resolve_bloom_filters(cfg, SCHEMA) == [True, False, True, True, True, True]
    cfg = WriteConfig(column_options={"v": ColumnOptions(enable_bloom_filter=True), "t": ColumnOptions(enable_dict=True)})
    assert resolve_bloom_filters(cfg, SCHEMA) == [False, False, True, False, False, False]
    assert resolve_bloom_filters(WriteConfig(column_options={"v": ColumnOptions(enable_bloom_filter=False)}), SCHEMA) is None
    # the per-column writer options are unchanged by the bloom setting
    assert resolve_column_options(WriteConfig(enable_bloom_filter=True), SCHEMA) == resolve_column_options(WriteConfig(), SCHEMA)


def test_host_writer_writes_the_filters():
    st = StorageSchema.try_new(USER, 2)
    batch = record_batch(USER, {"k": [2, 1, 3], "ts": [5, 6, 7], "v": [0.5, None, 1.5], "t": [3, None, 4]})
    data = sstgen.write_sst(st, batch, 1, WriteConfig(column_options={"v": ColumnOptions(enable_bloom_filter=True)}))
    blooms = M.footer_blooms(data)
    assert [c for (g, c), e in blooms.items() if e["offset"] >= 0] == [2]
    nbytes, _, bits = M.read_filter(data, blooms[(0, 2)]["offset"])
    assert nbytes == 1 << 20 and bits == M.build(np.array([0.5, 1.5]).view(np.uint64), nbytes)
    assert "bloom_filter_options" not in sstgen._writer_kwargs(st, WriteConfig())


class _RecordingEngine:
    """Records the keyword arguments of the writer calls ObjectBasedStorage makes."""
    def __init__(self):
        self.calls = []

    def write_batch(self, schema, batch, sequence, out_path, **kw):
        self.calls.append(kw)
        with open(out_path, "wb") as f:
            f.write(b"")
        return _ffi.HgFileMeta(size=0, num_rows=batch.num_rows)


def test_storage_passes_bloom_filters_only_when_enabled(tmp_path):
    from horaedb_b200.storage import ObjectBasedStorage, WriteRequest
    from horaedb_b200.types import TimeRange
    batch = record_batch(USER, {"k": [2, 1], "ts": [5, 6], "v": [0.5, 1.5], "t": [3, None]})
    cases = [(WriteConfig(), None),
             (WriteConfig(column_options={"t": ColumnOptions(enable_bloom_filter=False)}), None),
             (WriteConfig(enable_bloom_filter=True), [True] * 6),
             (WriteConfig(enable_bloom_filter=True, column_options={"ts": ColumnOptions(enable_bloom_filter=False)}), [True, False, True, True, True, True])]
    for i, (cfg, want) in enumerate(cases):
        eng = _RecordingEngine()
        st = ObjectBasedStorage(str(tmp_path / str(i)), 1000, USER, 2, StorageConfig(write=cfg), engine=eng)
        st.write(WriteRequest(batch, TimeRange(0, 10)))
        assert len(eng.calls) == 1
        assert ("bloom_filters" in eng.calls[0]) == (want is not None), cfg
        if want is not None:
            assert eng.calls[0]["bloom_filters"] == want


def test_write_props_layout():
    import ctypes as C
    assert _ffi.HgColumnWriteOpts.bloom_filter.offset == 3 and C.sizeof(_ffi.HgColumnWriteOpts) == 4
    assert _ffi.HgWriteProps.bloom_filter_bytes.offset == 12 and C.sizeof(_ffi.HgWriteProps) == 24
    assert C.sizeof(_ffi.HgParquetBloom) == 32
    p = _ffi._write_props(8192, "zstd", True, None, [False, True], 4096)
    assert p.bloom_filter_bytes == 4096 and [(p.columns[i].codec, p.columns[i].bloom_filter) for i in range(2)] == [(6, 0), (6, 1)]
    assert not _ffi._write_props(8192, "snappy", True, None).columns
