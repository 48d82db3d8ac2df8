"""Every page decoder on encodings laid out the way other Parquet writers lay them out (tests/page_encodings.py): SSTs pyarrow wrote with
PLAIN values and no compression, their pages re-encoded, read by the engine and compared bit for bit with the C oracle on the source file.
The layouts make the choices pyarrow never makes: DELTA_BINARY_PACKED block / miniblock geometries from 128/1 to 4096/64, widths wider
than needed, junk in unused widths and padding bits, INT32 deltas in 64-bit arithmetic; dictionary indices in RLE-only, bit-packed-only
and alternating runs, wide index widths, width 0, PLAIN_DICTIONARY ids, a fallback to PLAIN mid-chunk, a dictionary page no offset
names; definition levels in any run split; pages of 1 and 7 rows; one chunk mixing DELTA, PLAIN and dictionary pages; on Binary columns,
DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY pages whose length runs take the DELTA layouts, and Binary dictionaries.  Covered: scan
(merge, dedup, batch boundaries, resident and transient, every fixed-width type with NULLs) with the chunk statistics kept (null_count
= 0 chunks get no validity buffer) and stripped, RUNS / HASH aggregates, compaction, the fused Snappy aggregate and both row-group
gates on level layouts, stored pages, one range function per family, and the refusal of deprecated BIT_PACKED levels."""
import functools
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import foreign_streams as fs
import page_encodings as pe
import page_recode as pr
from helpers import arrays_equal, check_stream
from horaedb_b200 import sstgen
from horaedb_b200._ffi import (HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_LATE_MATERIALIZATION, HG_FN_RATE, Engine, HgError,
                               SchemaHandle, SstInput)
from horaedb_b200.config import WriteConfig
from horaedb_b200.types import StorageSchema
from oracle import oracle
from range_function_model import range_function

pytestmark = pytest.mark.gpu
_ids = iter(range(120_000_000, 130_000_000))
T0 = sstgen.T0_MS
METRIC = sstgen.metric_storage_schema()
ALL_TYPES = ("uint8", "int8", "uint16", "int16", "uint32", "int32", "uint64", "int64", "float32", "float64")


# ---- source files: PLAIN, no dictionary, uncompressed

def _write(schema, batch, seq, rg, v2):
    full = schema.fill_builtin_columns(batch, seq)
    kw = sstgen._writer_kwargs(schema, WriteConfig(compression="none", max_row_group_size=rg))
    kw["data_page_version"] = "2.0" if v2 else "1.0"
    sink = io.BytesIO()
    pq.write_table(pa.Table.from_batches([full]), sink, **kw)
    return sink.getvalue()


@functools.lru_cache(maxsize=None)
def metric_src(lo, nseries, points, seq, nulls=0.0, rg=1024, v2=False):
    """series [lo, lo + nseries), `points` samples each; tag = series mod 16; value random with a share of NULLs"""
    rng = np.random.default_rng(seq)
    sid = np.repeat(np.arange(lo, lo + nseries, dtype=np.uint64), points)
    n = len(sid)
    ts = T0 + np.tile(np.arange(points, dtype=np.int64) * 1000, nseries) + rng.integers(0, 500, n)
    v = rng.random(n) * 100 - 20
    mask = rng.random(n) < nulls if nulls else None
    batch = pa.RecordBatch.from_arrays([pa.array(sid), pa.array(ts), pa.array(v, mask=mask), pa.array((sid % 16).astype(np.uint32))],
                                       schema=sstgen.METRIC_SCHEMA)
    return _write(METRIC, batch, seq, rg, v2)


def all_types_schema():
    fields = [pa.field("series_id", pa.uint64(), True), pa.field("ts", pa.int64(), True)]
    fields += [pa.field(f"c_{t}", getattr(pa, t)(), True) for t in ALL_TYPES]
    schema = StorageSchema.try_new(pa.schema(fields), 2)
    schema.user_arrow = pa.schema(fields)
    return schema


@functools.lru_cache(maxsize=None)
def all_types_src(v2=False):
    """every fixed-width type, 10 % NULLs, small-range and full-range values; the 64-bit columns start with the extremes in turn"""
    rng = np.random.default_rng(7)
    schema = all_types_schema()
    n = 1500
    cols = [pa.array(np.repeat(np.arange(15, dtype=np.uint64), 100)), pa.array(T0 + np.tile(np.arange(100) * 1000, 15))]
    for i, t in enumerate(ALL_TYPES):
        dt = np.dtype(t)
        if dt.kind == "f":
            v = np.round(rng.random(n) * 1000, 1 if i % 2 else 6).astype(dt)
        else:
            info = np.iinfo(dt)
            v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True) if i % 2 else rng.integers(0, 20, n).astype(dt)
            if dt.itemsize == 8:
                v[:16] = np.where(np.arange(16) % 2 == 0, info.min, info.max).astype(dt)
        mask = rng.random(n) < 0.1
        if dt.itemsize == 8:
            mask[:16] = False
        cols.append(pa.array(v, mask=mask))
    batch = pa.RecordBatch.from_arrays(cols, schema=schema.user_arrow)
    return _write(schema, batch, 77, 1000, v2)


def binary_schema():
    fields = [pa.field("series_id", pa.uint64(), True), pa.field("ts", pa.int64(), True), pa.field("blob", pa.binary(), True),
              pa.field("name", pa.binary(), True)]
    schema = StorageSchema.try_new(pa.schema(fields), 2)
    schema.user_arrow = pa.schema(fields)
    return schema


@functools.lru_cache(maxsize=None)
def binary_src(v2=False):
    """two Binary columns: `blob` with 15 % NULLs, lengths 0 to 40 (some 300) over a few shared prefixes; `name` without NULLs (its chunks
    null_count = 0), one of five strings"""
    rng = np.random.default_rng(17)
    n = 1500
    prefixes = [b"", b"cpu.", b"cpu.user.", b"mem.heap.", bytes(range(200, 220))]
    blob = []
    for i in range(n):
        tail = rng.integers(0, 256, int(rng.integers(0, 24)), dtype=np.uint8).tobytes()
        v = prefixes[int(rng.integers(0, len(prefixes)))] + tail
        blob.append(v * 10 if i % 97 == 5 else v)
    mask = rng.random(n) < 0.15
    names = [b"host-a", b"host-b", b"", b"host-c-long-name", b"x"]
    cols = [pa.array(np.repeat(np.arange(15, dtype=np.uint64), 100)), pa.array(T0 + np.tile(np.arange(100) * 1000, 15)),
            pa.array(blob, pa.binary(), mask=mask), pa.array([names[int(k)] for k in rng.integers(0, 5, n)], pa.binary())]
    schema = binary_schema()
    return _write(schema, pa.RecordBatch.from_arrays(cols, schema=schema.user_arrow), 78, 1000, v2)


def overlapping_sources():
    """three overlapping files, V1 and V2 pages; the value column has NULLs, every other column null_count = 0 (__reserved__: all NULL)"""
    return [metric_src(lo, 8, 200, seq, nulls=0.05, v2=seq == 2) for seq, lo in ((1, 0), (2, 3), (3, 6))]


# ---- layouts: name -> encode(chunk, feats) -> [Page] (None: the source's pages)

def _int_col(c):
    return c.phys in (pe.INT32, pe.INT64)


def delta_layout(block, nmini, extra=0, junk=False, arith64=False):
    """integer columns: DELTA_BINARY_PACKED pages; Binary columns: DELTA_LENGTH_BYTE_ARRAY and DELTA_BYTE_ARRAY pages in turn, whose
    length runs take the same geometry, widths and padding"""
    def enc(c, feats):
        opts = dict(block=block, nmini=nmini, extra=extra, junk=junk, arith64=arith64)
        pages = []
        if c.phys == pe.BYTE_ARRAY:
            for k, (a, b) in enumerate(pe.split_rows(c, [1, block, block + 1, 700])):
                vals = pe.values_in(c, a, b)
                dba = k % 2 == 1
                pages.append(pe.Page(rows=b - a, encoding=pe.DBA if dba else pe.DLBA,
                                     values=(pe.dba_encode if dba else pe.dlba_encode)(vals, feats, **opts)))
            return pages
        if not _int_col(c):
            return None
        bits = 32 if c.phys == pe.INT32 else 64
        for a, b in pe.split_rows(c, [1, block, block + 1, 700]):
            vals = pe.signed(c, pe.values_in(c, a, b))
            pages.append(pe.Page(rows=b - a, encoding=pe.DELTA, values=pe.delta_encode(vals, bits, feats=feats, **opts)))
        return pages
    return enc


def dictionary_of(c):
    uniq = list(dict.fromkeys(c.values))
    return uniq, {v: i for i, v in enumerate(uniq)}


def dict_layout(style="arrow", extra=0, ids=pe.RLE_DICT, fallback_after=None, named=True, pad_ones=False, sizes=(333, 700)):
    def enc(c, feats):
        uniq, idx = dictionary_of(c)
        w = min(32, (len(uniq) - 1).bit_length() + extra) if uniq else 0
        feats[f"index_width_{w}"] = feats.get(f"index_width_{w}", 0) + 1
        if w == 0 and len(uniq) == 1:
            feats["width_0_one_entry"] = feats.get("width_0_one_entry", 0) + 1
        if w > 24:
            feats["index_width_over_24"] = feats.get("index_width_over_24", 0) + 1
        if c.phys == pe.BYTE_ARRAY:
            feats["binary_dictionary"] = feats.get("binary_dictionary", 0) + 1
        pages = [pe.Page(rows=len(uniq), values=pe.plain(c, uniq), dictionary=True, encoding=pe.PLAIN_DICT if ids == pe.PLAIN_DICT else pe.PLAIN,
                         named=named)]
        if not named:
            feats["dictionary_page_unnamed"] = feats.get("dictionary_page_unnamed", 0) + 1
        for k, (a, b) in enumerate(pe.split_rows(c, list(sizes))):
            vals = pe.values_in(c, a, b)
            if fallback_after is not None and k >= fallback_after:
                pages.append(pe.Page(rows=b - a, values=pe.plain(c, vals)))
                feats["fallback_to_plain"] = feats.get("fallback_to_plain", 0) + 1
                continue
            body = bytes([w]) + pe.hybrid_encode([idx[v] for v in vals], w, style, feats, seed=a, pad=(1 << w) - 1 if pad_ones else 0)
            pages.append(pe.Page(rows=b - a, values=body, encoding=ids))
            if ids == pe.PLAIN_DICT:
                feats["plain_dictionary_ids"] = feats.get("plain_dictionary_ids", 0) + 1
        return pages
    return enc


def levels_layout(style):
    """one PLAIN V1 page per chunk, its definition levels in the given run split"""
    def enc(c, feats):
        if not c.optional:
            return None
        if c.null_count_zero:
            feats["all_valid_chunk"] = feats.get("all_valid_chunk", 0) + 1
        return [pe.Page(rows=len(c.levels), values=pe.plain(c, c.values), levels=pe.hybrid_encode(c.levels, 1, style, feats), v2=False)]
    return enc


def pages_1_7(c, feats):
    feats["pages_of_1_and_7"] = feats.get("pages_of_1_and_7", 0) + 1
    return [pe.Page(rows=b - a, values=pe.plain(c, pe.values_in(c, a, b))) for a, b in pe.split_rows(c, [1, 7] * 6 + [500])]


def mixed(c, feats):
    """a dictionary page, then DELTA, PLAIN and dictionary pages in turn"""
    if not _int_col(c):
        return None
    uniq, idx = dictionary_of(c)
    w = (len(uniq) - 1).bit_length() if uniq else 0
    bits = 32 if c.phys == pe.INT32 else 64
    pages = [pe.Page(rows=len(uniq), values=pe.plain(c, uniq), dictionary=True)]
    for k, (a, b) in enumerate(pe.split_rows(c, [100, 37, 260, 129, 300])):
        vals = pe.values_in(c, a, b)
        kind = k % 3
        if kind == 0:
            pages.append(pe.Page(rows=b - a, encoding=pe.DELTA, values=pe.delta_encode(pe.signed(c, vals), bits, 256, 8, feats=feats)))
        elif kind == 1:
            pages.append(pe.Page(rows=b - a, values=pe.plain(c, vals)))
        else:
            pages.append(pe.Page(rows=b - a, encoding=pe.RLE_DICT, values=bytes([w]) + pe.hybrid_encode([idx[v] for v in vals], w, "alternate", feats, a)))
    feats["mixed_chunk"] = feats.get("mixed_chunk", 0) + 1
    return pages


LAYOUTS = {
    "delta_128_1": delta_layout(128, 1), "delta_256_8": delta_layout(256, 8), "delta_256_2": delta_layout(256, 2),
    "delta_1024_8": delta_layout(1024, 8), "delta_2048_16": delta_layout(2048, 16), "delta_4096_64": delta_layout(4096, 64),
    "delta_wide": delta_layout(128, 4, extra=64), "delta_junk": delta_layout(128, 4, junk=True),
    "delta_i32_64bit": delta_layout(128, 4, arith64=True),
    "dict_rle": dict_layout("rle"), "dict_packed": dict_layout("packed", sizes=(2000,)), "dict_alternate": dict_layout("alternate"),
    "dict_mod8": dict_layout("mod8"), "dict_wide": dict_layout("arrow", extra=32), "dict_wide_23": dict_layout("alternate", extra=11),
    "dict_plain_dictionary": dict_layout("arrow", ids=pe.PLAIN_DICT), "dict_fallback": dict_layout("arrow", fallback_after=1, sizes=(300,)),
    "dict_unnamed": dict_layout("rle", named=False), "dict_pad_ones": dict_layout("packed", extra=1, pad_ones=True, sizes=(77, 333)),
    "levels_rle": levels_layout("rle"), "levels_short_rle": levels_layout("short_rle"), "levels_packed": levels_layout("packed"),
    "levels_alternate": levels_layout("alternate"), "levels_mod8": levels_layout("mod8"),
    "pages_1_7": pages_1_7, "mixed": mixed,
}
LEVEL_NAMES = [n for n in LAYOUTS if n.startswith("levels_")]
# layouts pyarrow 24 refuses to read (checked in tests/test_oracle_foreign_encodings.py); their expected rows are the source's
PYARROW_REFUSES = {"delta_i32_64bit"}


@functools.lru_cache(maxsize=None)
def recoded(src, name, drop_stats=False):
    """(the source re-laid out by LAYOUTS[name], the features the layout emitted, summed)"""
    feats = {}
    ncols = pq.ParquetFile(io.BytesIO(src)).metadata.num_columns
    out = pe.recode(src, lambda c: LAYOUTS[name](c, feats), pyarrow_reads=name not in PYARROW_REFUSES,
                    drop_stats=range(2, ncols) if drop_stats else ())           # (the primary keys keep theirs: they must not be NULL)
    return out, feats


def _inputs(eng, handle, datas, resident):
    ins = []
    for d in datas:
        i = next(_ids)
        if resident:
            eng.load_sst(handle, SstInput(id=i, data=d))
            ins.append(SstInput(id=i, num_rows=pq.ParquetFile(io.BytesIO(d)).metadata.num_rows))
        else:
            ins.append(SstInput(id=i, data=d))
    return ins


def _check_agg(got, exp, bucket):
    assert got.num_rows == len(exp.count)
    if got.num_rows:
        assert got["series_id"].to_numpy().tolist() == exp.gkey.tolist()
        if bucket:
            assert got["bucket"].to_numpy().tolist() == exp.bucket.tolist()
        assert got["count"].to_numpy().tolist() == exp.count.tolist()
        for c in ("sum", "min", "max"):
            assert got[c].to_numpy().tobytes() == getattr(exp, c).tobytes(), c


KW = dict(group_col=0, ts_col=1, window_ms=60_000, value_col=2)
KW_SERIES = dict(group_col=0, ts_col=-1, window_ms=0, value_col=2)
PREDS = [("tag", "eq", 3), ("ts", "ge", T0 + 20_000), ("ts", "lt", T0 + 150_000)]


# ---- scan: merge, dedup, batch boundaries; every fixed-width type

@pytest.mark.parametrize("stats", ["kept", "stripped"])
@pytest.mark.parametrize("name", list(LAYOUTS))
def test_scan_recoded(name, stats):
    drop = stats == "stripped"
    srcs = overlapping_sources()
    datas = [recoded(s, name, drop)[0] for s in srcs]
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    for resident, batch_size in ((True, 8192), (False, 500)):
        eng = Engine(device=0, batch_size=batch_size)
        ins = _inputs(eng, handle, datas, resident)
        for preds in ([], [("tag", "eq", 3), ("ts", "ge", T0 + 50_000)]):
            got = list(eng.scan(handle, ins, preds))
            check_stream(got, oracle.scan(srcs, METRIC.arrow_schema, 2, preds, batch_size=batch_size).batches)
        eng.close()
    for v2 in (False, True):
        src = all_types_src(v2)
        data = recoded(src, name, drop)[0]
        schema = all_types_schema()
        handle = SchemaHandle(schema.arrow_schema, 2)
        eng = Engine(device=0)
        got = eng.scan(handle, _inputs(eng, handle, [data], False)).read_all()
        eng.close()
        exp = oracle.decode_sst(src, schema.arrow_schema)
        ref = pq.read_table(io.BytesIO(src))
        assert got.num_rows == exp.num_rows == ref.num_rows
        for c in schema.user_arrow.names:
            assert arrays_equal(got[c], exp[c]) and arrays_equal(got[c], ref[c]), c


@pytest.mark.parametrize("stats", ["kept", "stripped"])
@pytest.mark.parametrize("name", list(LAYOUTS))
def test_scan_binary_recoded(name, stats):
    """Binary columns with and without NULLs, V1 and V2 pages: DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY pages whose length runs take
    every DELTA layout (where the bytes behind a run start is decided by the run's end), the dictionary index layouts on Binary entries,
    the level layouts and the page splits; resident and transient, against pyarrow on the source"""
    schema = binary_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    for v2 in (False, True):
        src = binary_src(v2)
        data = recoded(src, name, stats == "stripped")[0]
        ref = pq.read_table(io.BytesIO(src))
        for resident in (True, False):
            eng = Engine(device=0)
            got = eng.scan(handle, _inputs(eng, handle, [data], resident)).read_all()
            eng.close()
            assert got.num_rows == ref.num_rows
            for c in schema.user_arrow.names:
                assert arrays_equal(got[c], ref[c]), (c, v2, resident)


# ---- RUNS / HASH aggregates on the general pipeline, compaction

@pytest.mark.parametrize("name", list(LAYOUTS))
def test_aggregate_recoded(name):
    srcs = overlapping_sources()
    datas = [recoded(s, name)[0] for s in srcs]
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    eng = Engine(device=0)
    for mode in (HG_AGG_RUNS, HG_AGG_HASH):
        for resident in (True, False):
            got = eng.scan_aggregate(handle, _inputs(eng, handle, datas, resident), PREDS, mode=mode, **KW)
            _check_agg(got, oracle.scan_aggregate(srcs, METRIC.arrow_schema, 2, PREDS, mode=mode, **KW), True)
    eng.close()


@pytest.mark.parametrize("name", ["delta_4096_64", "delta_junk", "dict_packed", "dict_unnamed", "levels_alternate", "mixed"])
def test_compact_recoded(name, tmp_path):
    srcs = overlapping_sources()
    datas = [recoded(s, name)[0] for s in srcs]
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    eng = Engine(device=0)
    got = eng.compact(handle, _inputs(eng, handle, datas, False)).read_all()
    exp = eng.compact(handle, _inputs(eng, handle, srcs, False)).read_all()
    assert got.equals(exp)
    out = str(tmp_path / "c.sst")
    eng.compact_to_sst(handle, _inputs(eng, handle, datas, False), out)
    eng.close()
    back = pq.read_table(out)
    assert back.num_rows == exp.num_rows
    for c in exp.column_names:
        assert arrays_equal(back[c], exp[c]), c


# ---- level layouts on Snappy pages: the fused aggregate, both row-group gates, stored pages

def _snappy(data, literal_only=False):
    """`data` with every page Snappy-compressed: by libsnappy, or as one literal (a page 4+ bytes per row: the gate column is
    decompressed first and gate_rgs_kernel reads it)"""
    comp = (lambda raw, ci, pn: fs.snappy_literals_split(raw, [])[0]) if literal_only else \
        (lambda raw, ci, pn: pa.Codec("snappy").compress(raw, asbytes=True))
    return pr.recode(data, comp, pr.SNAPPY)


def fused_source():
    """no NULLs: the fused aggregate takes every chunk (null_count = 0)"""
    return metric_src(0, 20, 600, 11, rg=4000)


@pytest.mark.parametrize("literal_only", [False, True])
@pytest.mark.parametrize("name", LEVEL_NAMES)
def test_fused_and_gate_on_level_layouts(name, literal_only):
    """The benchmark's shape on the level layouts: the fused path (with and without late materialisation) gives the oracle's result on
    the source.  The gate on tag takes its bits from the Snappy stream (two launches more than the ungated call) for libsnappy pages,
    and from the decompressed page by gate_rgs_kernel (three more) for pages stored as one literal."""
    src = fused_source()
    data = _snappy(recoded(src, name)[0], literal_only)
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    for preds, kw in ((PREDS, KW), (PREDS, KW_SERIES), ([("tag", "eq", 3)], KW)):
        exp = oracle.scan_aggregate([src], METRIC.arrow_schema, 2, preds, **kw)
        for resident in (True, False):
            eng = Engine(device=0)
            got = eng.scan_aggregate(handle, _inputs(eng, handle, [data], resident), preds, **kw)
            assert eng.stats()["path"] & 1
            eng.close()
            _check_agg(got, exp, kw["ts_col"] >= 0)
    launches = []
    for flags in (0, HG_FLAG_NO_LATE_MATERIALIZATION):
        eng = Engine(device=0, flags=flags)
        got = eng.scan_aggregate(handle, _inputs(eng, handle, [data], True), [("tag", "eq", 3)], **KW)
        launches.append(eng.stats()["kernel_launches"])
        eng.close()
    md = pq.ParquetFile(io.BytesIO(data)).metadata
    stream_gate = sum(md.row_group(g).column(3).total_compressed_size for g in range(md.num_row_groups)) * 2 < md.num_rows
    assert stream_gate == (not literal_only)
    assert launches[0] == launches[1] + (2 if stream_gate else 3), launches


# ---- one range function per family

@pytest.mark.parametrize("name", ["delta_2048_16", "dict_mod8", "levels_packed", "pages_1_7", "mixed"])
def test_rate_on_recoded_files(name):
    srcs = [metric_src(lo, 6, 300, seq) for seq, lo in ((51, 0), (52, 6))]
    datas = [recoded(s, name)[0] for s in srcs]
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    grid = (T0 + 60_000, T0 + 290_000, 30_000, 60_000)
    exp = range_function(srcs, METRIC.arrow_schema, 2, HG_FN_RATE, [], *grid)
    eng = Engine(device=0)
    got = eng.scan_range_function(handle, _inputs(eng, handle, datas, False), HG_FN_RATE, [], *grid)
    eng.close()
    assert got.num_rows == exp.num_rows > 0
    assert got.column(0).to_pylist() == exp.column(0).to_pylist() and got["t"].to_pylist() == exp["t"].to_pylist()
    assert got["value"].to_numpy().tobytes() == exp["value"].to_numpy().tobytes()


# ---- deprecated BIT_PACKED levels

def bit_packed_levels(c, feats):
    """V1 pages whose definition levels are BIT_PACKED (no length in front of them)"""
    feats["bit_packed_levels"] = feats.get("bit_packed_levels", 0) + 1
    return [pe.Page(rows=len(c.levels), values=pe.plain(c, c.values), levels=pe.bit_packed_levels(c.levels) if c.optional else None,
                    level_encoding=pe.BIT_PACKED, v2=False)]


@functools.lru_cache(maxsize=None)
def required_src():
    """the metric schema with every column REQUIRED"""
    schema = pa.schema([f.with_nullable(False) for f in METRIC.arrow_schema], metadata=METRIC.arrow_schema.metadata)
    rng = np.random.default_rng(5)
    sid = np.repeat(np.arange(10, dtype=np.uint64), 100)
    n = len(sid)
    cols = [sid, T0 + np.tile(np.arange(100) * 1000, 10), rng.random(n), (sid % 16).astype(np.uint32), np.full(n, 9, np.uint64),
            np.zeros(n, np.uint64)]
    t = pa.Table.from_arrays([pa.array(c) for c in cols], schema=schema)
    sink = io.BytesIO()
    pq.write_table(t, sink, compression="none", use_dictionary=False, data_page_version="1.0", store_schema=True)
    return sink.getvalue()


def test_bit_packed_levels_refused_on_optional_columns():
    src = metric_src(0, 4, 100, 61, nulls=0.1)
    data = pe.recode(src, lambda c: bit_packed_levels(c, {}), pyarrow_reads=False)   # (pyarrow 24 reads these bits LSB first)
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    eng = Engine(device=0)
    with pytest.raises(HgError) as ei:
        eng.scan(handle, _inputs(eng, handle, [data], False)).read_all()
    eng.close()
    assert ei.value.code == 2, ei.value                                  # HG_ERR_UNSUPPORTED
    assert str(ei.value).endswith("column 0 (series_id): definition levels in the deprecated BIT_PACKED encoding (4); RLE levels are implemented"), str(ei.value)


def test_bit_packed_label_on_required_columns_is_read():
    src = required_src()
    data = pe.recode(src, lambda c: bit_packed_levels(c, {}))
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    eng = Engine(device=0)
    got = eng.scan(handle, _inputs(eng, handle, [data], False)).read_all()
    eng.close()
    ref = pq.read_table(io.BytesIO(src))
    assert got.num_rows == ref.num_rows
    for c in ("series_id", "ts", "value", "tag"):
        assert arrays_equal(got[c], ref[c]), c
