"""Every page path on Snappy and Zstandard streams from other encoders (tests/foreign_streams.py): SSTs written by pyarrow, their pages
rewritten with tests/page_recode.py, read by the engine and compared bit for bit with the C oracle on the source file (uncompressed, or
the libsnappy original).  The streams make the choices libsnappy and one-shot libzstd never make: copies across 64 KiB and with 4-byte
offsets, 1-3 byte copies, wide literal headers, literals split anywhere, streaming frames without content size, several frames per
page, skippable frames, checksums, raw / RLE blocks.  Covered: the general pipeline (merge, dedup, batch boundaries), the fused Snappy
aggregate with and without the gate bits taken from the stream, stored (literal-only) pages split at every row, compressed prefixes of
lopsided pages, Zstandard pages through scan / aggregate / compaction, and one range function per codec."""
import functools
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import foreign_streams as fs
import page_recode as pr
from helpers import arrays_equal, check_stream
from horaedb_b200 import sstgen
from horaedb_b200._ffi import (HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_FUSED, HG_FLAG_NO_LATE_MATERIALIZATION, HG_FN_RATE, Engine, SchemaHandle,
                               SstInput)
from horaedb_b200.config import ParquetCompression, WriteConfig
from horaedb_b200.types import StorageSchema
from oracle import oracle
from range_function_model import range_function

pytestmark = pytest.mark.gpu
_ids = iter(range(110_000_000, 120_000_000))
T0 = sstgen.T0_MS
METRIC = sstgen.metric_storage_schema()
ALL_TYPES = ("uint8", "int8", "uint16", "int16", "uint32", "int32", "uint64", "int64", "float32", "float64")


# ---- source files

@functools.lru_cache(maxsize=None)
def metric_src(lo, nseries, points, seq, nulls=0.0, rg=4096, compression=ParquetCompression.Uncompressed, value="random"):
    """series [lo, lo + nseries) with `points` samples each; tag = series mod 16 (runs); value random, or random for the first 40 % of
    each row group and constant after (`lopsided`), or repeating every 8 200 rows (`periodic`: matches 65 600 bytes back)"""
    rng = np.random.default_rng(seq)
    sid = np.repeat(np.arange(lo, lo + nseries, dtype=np.uint64), points)
    n = len(sid)
    ts = T0 + np.tile(np.arange(points, dtype=np.int64) * 1000, nseries) + rng.integers(0, 500, n)
    v = rng.random(n) * 100 - 20
    if value == "lopsided":
        v = np.where((np.arange(n) % rg) < rg * 2 // 5, v, 0.5)
    elif value == "periodic":
        v = np.resize(v[:8200], n)
    mask = rng.random(n) < nulls if nulls else None
    batch = pa.RecordBatch.from_arrays([pa.array(sid), pa.array(ts), pa.array(v, mask=mask), pa.array((sid % 16).astype(np.uint32))],
                                       schema=sstgen.METRIC_SCHEMA)
    return sstgen.write_sst(METRIC, batch, seq=seq, cfg=WriteConfig(compression=compression, max_row_group_size=rg), presorted=True)


def all_types_schema():
    fields = [pa.field("series_id", pa.uint64(), True), pa.field("ts", pa.int64(), True)]
    fields += [pa.field(f"c_{t}", getattr(pa, t)(), True) for t in ALL_TYPES]
    schema = StorageSchema.try_new(pa.schema(fields), 2)
    schema.user_arrow = pa.schema(fields)
    return schema


@functools.lru_cache(maxsize=None)
def all_types_src(seq=77):
    """every fixed-width type, 10 % NULLs, small-range and full-range values"""
    rng = np.random.default_rng(seq)
    schema = all_types_schema()
    n = 5000
    cols = [pa.array(np.repeat(np.arange(50, dtype=np.uint64), 100)), pa.array(T0 + np.tile(np.arange(100) * 1000, 50))]
    for i, t in enumerate(ALL_TYPES):
        dt = np.dtype(t)
        if dt.kind == "f":
            v = np.round(rng.random(n) * 1000, 1 if i % 2 else 6).astype(dt)
        else:
            info = np.iinfo(dt)
            v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True) if i % 2 else rng.integers(0, 20, n).astype(dt)
        cols.append(pa.array(v, mask=rng.random(n) < 0.1))
    batch = pa.RecordBatch.from_arrays(cols, schema=schema.user_arrow)
    return sstgen.write_sst(schema, batch, seq=seq, cfg=WriteConfig(compression=ParquetCompression.Uncompressed, max_row_group_size=3000),
                            presorted=True)


# ---- encoders: name -> (codec, compress(raw) -> (stream, counts))

ENCODERS = {name: (pr.SNAPPY, f) for name, f in fs.SNAPPY_ENCODERS.items()}
ENCODERS["lopsided"] = (pr.SNAPPY, lambda raw: fs.snappy_lopsided(raw, len(raw) * 3 // 5))
ENCODERS["literals_anywhere"] = (pr.SNAPPY, lambda raw: fs.snappy_literals_split(raw, [1, len(raw) // 3, len(raw) // 3 + 5, len(raw) - 1]))
ENCODERS.update({"zstd_" + name: (pr.ZSTD, lambda raw, f=f: (f(raw), {})) for name, f in fs.ZSTD_ENCODERS.items()})
SNAPPY_NAMES = [n for n, (c, _) in ENCODERS.items() if c == pr.SNAPPY]
ZSTD_NAMES = [n for n, (c, _) in ENCODERS.items() if c == pr.ZSTD]


@functools.lru_cache(maxsize=None)
def recoded(src, name):
    """(the source file with every page re-encoded by ENCODERS[name], the encoder's summed counts)"""
    codec, f = ENCODERS[name]
    total = {}

    def comp(raw, ci, pn):
        stream, counts = f(raw)
        for k, v in counts.items():
            total[k] = total.get(k, 0) + v
        return stream

    return pr.recode(src, comp, codec), total


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
BENCH_PREDS = [("tag", "eq", 3), ("ts", "ge", T0 + 50_000), ("ts", "lt", T0 + 300_000)]


# ---- general pipeline: merge, dedup and batch boundaries over three overlapping files

def _overlapping_sources():
    return [metric_src(lo, 12, 400, seq, nulls=0.05, rg=2048) for seq, lo in ((1, 0), (2, 5), (3, 10))]


@pytest.mark.parametrize("resident", [True, False])
@pytest.mark.parametrize("name", list(ENCODERS))
def test_scan_overlapping_recoded_files(name, resident):
    srcs = _overlapping_sources()
    datas = [recoded(s, name)[0] for s in srcs]
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    for batch_size in (8192, 1000):
        eng = Engine(device=0, batch_size=batch_size)
        ins = _inputs(eng, handle, datas, resident)
        for preds in ([], [("tag", "eq", 3), ("ts", "ge", T0 + 100_000)]):
            got = list(eng.scan(handle, ins, preds))
            check_stream(got, oracle.scan(srcs, METRIC.arrow_schema, 2, preds, batch_size=batch_size).batches)
        eng.close()


@pytest.mark.parametrize("name", list(ENCODERS))
def test_scan_all_types_recoded(name):
    """every fixed-width type with NULLs: the engine's columns equal pyarrow's reading of the recoded file and the oracle's of the source"""
    src = all_types_src()
    data, _ = recoded(src, name)
    schema = all_types_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    got = eng.scan(handle, _inputs(eng, handle, [data], False)).read_all()
    eng.close()
    ref = pq.read_table(io.BytesIO(data))
    exp = oracle.decode_sst(src, schema.arrow_schema)
    assert got.num_rows == ref.num_rows == exp.num_rows
    for c in schema.user_arrow.names:
        assert arrays_equal(got[c], ref[c]) and arrays_equal(got[c], exp[c]), c


# ---- the fused Snappy aggregate

def fused_sources():
    """libsnappy files: 8 192-row groups, and 20 000-row groups whose 160 KB value pages repeat every 65 600 bytes"""
    return [metric_src(0, 20, 500, 11, rg=8192, compression=ParquetCompression.Snappy),
            metric_src(20, 20, 1000, 12, rg=20_000, compression=ParquetCompression.Snappy, value="periodic")]

@pytest.mark.parametrize("resident", [True, False])
@pytest.mark.parametrize("name", SNAPPY_NAMES)
def test_fused_aggregate_recoded(name, resident):
    """the benchmark's shape (tag = 3 AND ts in [a, b), sum / count per series, with and without buckets) on libsnappy sources re-encoded:
    the fused path, also without late materialisation, and the general pipeline give the oracle's result on the source"""
    srcs = fused_sources()
    datas = [recoded(s, name)[0] for s in srcs]
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    for kw in (KW, KW_SERIES):
        exp = oracle.scan_aggregate(srcs, METRIC.arrow_schema, 2, BENCH_PREDS, **kw)
        for flags in (0, HG_FLAG_NO_LATE_MATERIALIZATION, HG_FLAG_NO_FUSED):
            eng = Engine(device=0, flags=flags)
            got = eng.scan_aggregate(handle, _inputs(eng, handle, datas, resident), BENCH_PREDS, **kw)
            assert eng.stats()["path"] & 1 == (0 if flags == HG_FLAG_NO_FUSED else 1), flags
            eng.close()
            _check_agg(got, exp, kw["ts_col"] >= 0)


@pytest.mark.parametrize("name", ["identity"] + SNAPPY_NAMES)
def test_gate_bits_from_recoded_stream(name):
    """A run-coded 4-byte gate column: the row-group gate takes its bits straight from the gate column's Snappy pages, two launches more
    than the ungated call.  The planner takes that path while the column has under half a compressed byte per row; the encoders that
    write it wider (short copies, many literals) get the gate column decompressed first, three launches.  The result never changes."""
    src = metric_src(0, 30, 1000, 21, rg=8192, compression=ParquetCompression.Snappy)
    data = src if name == "identity" else recoded(src, name)[0]
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    exp = oracle.scan_aggregate([src], METRIC.arrow_schema, 2, [("tag", "eq", 3)], **KW)
    launches, results = [], []
    for flags in (0, HG_FLAG_NO_LATE_MATERIALIZATION):
        eng = Engine(device=0, flags=flags)
        got = eng.scan_aggregate(handle, _inputs(eng, handle, [data], True), [("tag", "eq", 3)], **KW)
        st = eng.stats()
        eng.close()
        assert st["path"] == 1
        _check_agg(got, exp, True)
        launches.append(st["kernel_launches"])
        results.append(got)
    assert results[0].equals(results[1])
    md = pq.ParquetFile(io.BytesIO(data)).metadata
    runs = sum(md.row_group(g).column(3).total_compressed_size for g in range(md.num_row_groups)) * 2 < md.num_rows
    assert runs == (name in ("identity", "copy2_only", "copy4_everywhere", "one_window", "wide_literal_headers"))
    assert launches[0] == launches[1] + (2 if runs else 3), launches


# ---- stored pages: literal-only value pages split at chosen rows

ROWS = 3000                                                        # rows per row group: one 24 KiB value literal in libsnappy's output


def _split_points(prefix, case):
    w = 8
    return {"one_literal": [], "n0=0": [prefix], "n0=1": [prefix + w], "n0=rows/2": [prefix + w * ROWS // 2],
            "n0=rows-1": [prefix + w * (ROWS - 1)], "inside_prefix": [prefix - 2], "prefix_too_short": [2],
            "inside_value": [prefix + w * 100 + 3], "three_literals": [prefix + w * 10, prefix + w * 2000]}[case]


STORED = ("one_literal", "n0=0", "n0=1", "n0=rows/2", "n0=rows-1")
DECLINED = ("inside_prefix", "prefix_too_short", "inside_value", "three_literals")


def _stored_file(case):
    src = metric_src(0, 24, 500, 31, rg=ROWS, compression=ParquetCompression.Snappy)
    ident = pr.identity(src)
    counts = []

    def comp(raw, ci, pn):
        if ci != 2:
            return ident(raw, ci, pn)
        prefix = 4 + int.from_bytes(raw[:4], "little")
        assert len(raw) - prefix == 8 * ROWS
        stream, c = fs.snappy_literals_split(raw, _split_points(prefix, case), hdr=3 if case == "n0=1" else None)
        counts.append(c["literal"])
        return stream

    return src, pr.recode(src, comp), counts


@pytest.mark.parametrize("case", STORED[1:] + DECLINED)
def test_stored_page_splits(case):
    """Resident and transient, gated: every split gives the oracle's result; a transient call ships only the row windows of an accepted
    split's value column, as for the page of one literal, and the whole chunk or a prefix of it for a declined one"""
    src, data, counts = _stored_file(case)
    assert set(counts) == {3 if case == "three_literals" else 2}
    _, one, _ = _stored_file("one_literal")
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    preds = [("tag", "eq", 3), ("ts", "lt", T0 + 200_000)]         # rows 1500-1699 of the first row group
    h2d = {}
    for kw in (KW, KW_SERIES):
        exp = oracle.scan_aggregate([src], METRIC.arrow_schema, 2, preds, **kw)
        for resident in (True, False):
            for d, key in ((data, case), (one, "one_literal")):
                eng = Engine(device=0)
                got = eng.scan_aggregate(handle, _inputs(eng, handle, [d], resident), preds, **kw)
                st = eng.stats()
                eng.close()
                assert st["path"] & 1
                _check_agg(got, exp, kw["ts_col"] >= 0)
                if not resident:
                    h2d[key] = st["bytes_h2d"]
    if case in STORED:
        assert abs(h2d[case] - h2d["one_literal"]) <= 64, h2d          # a literal header and a range's slack
    else:
        assert h2d[case] > h2d["one_literal"] + 8 * 1000, h2d


# ---- compressed prefixes

@pytest.mark.parametrize("name", ["lopsided", "random_parse"])
def test_compressed_prefix_of_recoded_page(name):
    """A transient gated aggregate ships a Snappy page decoded up to the last passing row as a prefix of its stream, estimated from the
    page's average ratio.  A lopsided stream (literal front, copy tail) runs out before that row: the call repeats with whole pages
    (stats path bit 2).  Either way: the resident result and the oracle's."""
    src = metric_src(0, 20, 1000, 41, rg=8192, compression=ParquetCompression.Snappy, value="lopsided")
    data, counts = recoded(src, name)
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    # passing rows only in the first third of every row group (series 3 and 19 of 20, 1000 rows each)
    preds = [("tag", "eq", 3)]
    exp = oracle.scan_aggregate([src], METRIC.arrow_schema, 2, preds, **KW_SERIES)
    res = {}
    for resident in (True, False):
        eng = Engine(device=0)
        res[resident] = eng.scan_aggregate(handle, _inputs(eng, handle, [data], resident), preds, **KW_SERIES)
        res[resident, "path"] = eng.stats()["path"]
        eng.close()
        _check_agg(res[resident], exp, False)
    assert res[True].equals(res[False])
    if name == "lopsided":
        assert res[False, "path"] & 2, res[False, "path"]          # the prefix ran out: the call was repeated with whole pages


# ---- Zstandard pages

@pytest.mark.parametrize("name", ZSTD_NAMES)
def test_zstd_recoded_aggregate_and_compact(name, tmp_path):
    srcs = _overlapping_sources()
    datas = [recoded(s, name)[0] for s in srcs]
    handle = SchemaHandle(METRIC.arrow_schema, 2)
    eng = Engine(device=0)
    for mode in (HG_AGG_RUNS, HG_AGG_HASH):
        for resident in (True, False):
            got = eng.scan_aggregate(handle, _inputs(eng, handle, datas, resident), BENCH_PREDS, mode=mode, **KW)
            _check_agg(got, oracle.scan_aggregate(srcs, METRIC.arrow_schema, 2, BENCH_PREDS, mode=mode, **KW), True)
    got = eng.compact(handle, _inputs(eng, handle, datas, False)).read_all()
    exp = eng.compact(handle, _inputs(eng, handle, srcs, False)).read_all()
    assert got.equals(exp)
    out = str(tmp_path / "c.sst")
    eng.compact_to_sst(handle, _inputs(eng, handle, datas, False), out, compression="zstd")
    eng.close()
    back = pq.read_table(out)
    assert back.num_rows == exp.num_rows
    for c in exp.column_names:
        assert arrays_equal(back[c], exp[c]), c


# ---- one analytic call per codec

@pytest.mark.parametrize("name", ["one_window", "short_copies", "zstd_stream_flush_1k", "zstd_raw_rle"])
def test_rate_on_recoded_files(name):
    srcs = [metric_src(lo, 10, 300, seq) for seq, lo in ((51, 0), (52, 10))]
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
