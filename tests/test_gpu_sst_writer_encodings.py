"""GPU SST writer with per-column writer options (hg_write_props.columns: csrc/sst_writer.cu delta_encode_kernel / dict_encode_kernel):
DELTA_BINARY_PACKED and dictionary pages with a codec per column, as parquet-rs writes them for a WriteConfig with `encoding`,
`enable_dict` or `column_options`.  The files must be SSTs of the reference's format — read by pyarrow, the CPU oracle and the GPU
engine — whose chunks carry the requested encodings and codecs, and whose pages hold what parquet-rs would put there: DELTA blocks of
128 with 4 miniblocks, dictionaries in first-appearance order keyed by the physical bits."""
import hashlib
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import Engine, HgError, SchemaHandle, SstInput
from horaedb_b200.config import ColumnOptions, ParquetEncoding, WriteConfig, resolve_column_options
from horaedb_b200.types import StorageSchema
from oracle import oracle

from helpers import arrays_equal, arrow_schema, record_batch

pytestmark = pytest.mark.gpu
_ids = iter(range(93_000_000, 96_000_000))
D, P = ParquetEncoding.DeltaBinaryPacked, ParquetEncoding.Plain

# SHA-256 of the file of test_mixed_output_is_pinned (same rows, options and row-group size -> same bytes, on the GPU and emulated)
PINNED_SHA256 = "4b94d66d9bd3c8a9909cd5b84c5e19be23dc7b9818350f2cf3c863cb2ed8e8b2"

# the three configurations of the metric schema (series_id, ts, value, tag, __seq__, __reserved__)
CONFIGS = {
    "delta_ints": WriteConfig(encoding=D, column_options={"value": ColumnOptions(encoding=P)}),
    "dict_all": WriteConfig(enable_dict=True),
    "mixed": WriteConfig(column_options={"series_id": ColumnOptions(enable_dict=True, compression="zstd"),
                                         "ts": ColumnOptions(encoding=D, compression="snappy"), "value": ColumnOptions(compression="snappy"),
                                         "tag": ColumnOptions(enable_dict=True), "__seq__": ColumnOptions(encoding=D, compression="none")},
                         compression="none"),
}


def _inputs(datas):
    return [SstInput(id=next(_ids), data=d, time_start=10 * i, time_end=10 * i + 5, max_sequence=100 + i) for i, d in enumerate(datas)]


# ---- a few lines of Thrift compact and Parquet page parsing -----------------------------------------------------------------------
def _uvarint(b, p):
    v = sh = 0
    while True:
        x = b[p]
        p += 1
        v |= (x & 0x7F) << sh
        sh += 7
        if not x & 0x80:
            return v, p


def _skip(b, p, t):
    if t in (1, 2):
        return p
    if t == 3:
        return p + 1
    if t in (4, 5, 6):
        return _uvarint(b, p)[1]
    if t == 7:
        return p + 8
    if t == 8:
        n, p = _uvarint(b, p)
        return p + n
    if t in (9, 10):
        h = b[p]
        p += 1
        n = h >> 4
        if n == 15:
            n, p = _uvarint(b, p)
        for _ in range(n):
            p = _skip(b, p, h & 15)
        return p
    assert t == 12, t
    return _struct(b, p)[1]


def _struct(b, p):
    """{field id: int value (i32 / i64) or nested dict} of one compact struct; other types are skipped."""
    out, last = {}, 0
    while True:
        h = b[p]
        p += 1
        if h == 0:
            return out, p
        t, d = h & 15, h >> 4
        if d:
            fid = last + d
        else:
            z, p = _uvarint(b, p)
            fid = (z >> 1) ^ -(z & 1)
        last = fid
        if t in (5, 6):
            z, p = _uvarint(b, p)
            out[fid] = (z >> 1) ^ -(z & 1)
        elif t == 12:
            out[fid], p = _struct(b, p)
        else:
            p = _skip(b, p, t)


_CODEC = {"UNCOMPRESSED": None, "SNAPPY": pa.Codec("snappy"), "ZSTD": pa.Codec("zstd")}


def _chunk_pages(data, col_md):
    """[(page type, header dict, decompressed payload)] of one column chunk (0 = data page, 2 = dictionary page)."""
    start = col_md.dictionary_page_offset if col_md.has_dictionary_page else col_md.data_page_offset
    end, p, out = start + col_md.total_compressed_size, start, []
    codec = _CODEC[col_md.compression]
    while p < end:
        h, q = _struct(data, p)
        raw = data[q:q + h[3]]
        out.append((h[1], h, raw if codec is None else codec.decompress(raw, decompressed_size=h[2], asbytes=True)))
        assert len(out[-1][2]) == h[2]
        p = q + h[3]
    assert p == end
    return out


def _levels_end(page):
    return 4 + int.from_bytes(page[:4], "little")


def _delta_widths(stream, pw):
    """Checks a DELTA_BINARY_PACKED stream's header (128 / 4) and returns (value count, bit widths of the stored miniblocks, bytes)."""
    block, p = _uvarint(stream, 0)
    mini, p = _uvarint(stream, p)
    count, p = _uvarint(stream, p)
    _, p = _uvarint(stream, p)
    assert (block, mini) == (128, 4)
    left, widths = max(count - 1, 0), []
    while left > 0:
        _, p = _uvarint(stream, p)
        bws = stream[p:p + 4]
        p += 4
        for m in range(4):
            if left > 0:
                assert bws[m] <= 8 * pw
                widths.append(bws[m])
                p += 4 * bws[m]
                left -= min(32, left)
            else:
                assert bws[m] == 0
    return count, widths, p


def _phys_bits(arr, pa_type):
    """The physical bits of the non-null values (1- / 2-byte integers widen to INT32, as the Parquet writer stores them)."""
    a = arr.drop_null() if hasattr(arr, "drop_null") else arr.filter(arr.is_valid())
    x = a.to_numpy(zero_copy_only=False)
    if pa.types.is_floating(pa_type):
        return x.view(np.uint64 if pa_type == pa.float64() else np.uint32)
    if pa_type.bit_width <= 32:
        return x.astype(np.int64 if pa.types.is_signed_integer(pa_type) else np.uint64).astype(np.int32 if pa.types.is_signed_integer(pa_type) else np.uint32).view(np.uint32)
    return x.view(np.uint64)


def _first_appearance(bits):
    _, first = np.unique(bits, return_index=True)
    return bits[np.sort(first)]


def _check_chunks(data, table, columns, rg):
    """Every chunk carries the requested encodings / dictionary / codec; DELTA headers and bit widths, dictionary pages = the chunk's
    first-appearance values, bit for bit."""
    md = pq.ParquetFile(io.BytesIO(data)).metadata
    names = table.schema.names
    for g in range(md.num_row_groups):
        lo = g * rg
        for c, name in enumerate(names):
            enc, dictionary, codec = columns[c]
            col = md.row_group(g).column(c)
            assert col.compression == {"none": "UNCOMPRESSED", "uncompressed": "UNCOMPRESSED"}.get(codec, codec.upper()), (g, name)
            part = table[name].combine_chunks().slice(lo, col.num_values)
            t = table.schema.field(name).type
            pw = 8 if t.bit_width == 64 else 4
            pages = _chunk_pages(data, col)
            if dictionary:
                assert col.has_dictionary_page and set(col.encodings) == {"PLAIN", "RLE", "RLE_DICTIONARY"}, (g, name, col.encodings)
                assert [pt for pt, _, _ in pages] == [2, 0]
                dpage = pages[0][2]
                want = _first_appearance(_phys_bits(part, t))
                assert pages[0][1][7][1] == len(want) and dpage == want.tobytes(), (g, name)
                assert pages[1][1][5][2] == 8                                         # RLE_DICTIONARY data page
            else:
                assert not col.has_dictionary_page and [pt for pt, _, _ in pages] == [0]
                if enc == D:
                    assert set(col.encodings) == {"RLE", "DELTA_BINARY_PACKED"}, col.encodings
                    assert pages[0][1][5][2] == 5
                    body = pages[0][2]
                    count, widths, used = _delta_widths(body[_levels_end(body):], pw)
                    assert count == len(part) - part.null_count and _levels_end(body) + used == len(body)
                else:
                    assert set(col.encodings) == {"PLAIN", "RLE"} and pages[0][1][5][2] == 0


def _expected_stats(plain, data):
    """Statistics of the encoded file equal those of the PLAIN output of the same rows."""
    a, b = pq.ParquetFile(io.BytesIO(plain)).metadata, pq.ParquetFile(io.BytesIO(data)).metadata
    assert a.num_row_groups == b.num_row_groups
    for g in range(a.num_row_groups):
        for c in range(a.num_columns):
            sa, sb = a.row_group(g).column(c).statistics, b.row_group(g).column(c).statistics
            assert sa.null_count == sb.null_count and sa.has_min_max == sb.has_min_max
            if sa.has_min_max:
                assert repr(sa.min) == repr(sb.min) and repr(sa.max) == repr(sb.max), (g, c)


def _read_equals(data, exp):
    got = pq.read_table(io.BytesIO(data))
    assert got.schema.names == exp.schema.names
    for name in exp.schema.names:
        assert got[name].type == exp[name].type and arrays_equal(got[name], exp[name]), name


@pytest.mark.parametrize("rg", [8192, 1000, 97])
@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_encoded_compaction_round_trips(tmp_path, cfg, rg):
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    datas = [s[0] for s in sstgen.synth_overlapping_ssts(5, series=24, points=300, delta_ms=1000, keep_frac=0.5, compression="snappy")]
    exp = pa.Table.from_batches(oracle.scan(datas, schema.arrow_schema, 2, (), True, 8192).batches)
    columns = resolve_column_options(CONFIGS[cfg], schema.arrow_schema)
    eng = Engine(device=0)
    path, plain = str(tmp_path / "enc.sst"), str(tmp_path / "plain.sst")
    meta = eng.compact_to_sst(handle, _inputs(datas), path, max_row_group_size=rg, columns=columns)
    eng.compact_to_sst(handle, _inputs(datas), plain, max_row_group_size=rg, compression="none")
    data = open(path, "rb").read()
    assert meta.size == len(data) and meta.num_rows == exp.num_rows
    _read_equals(data, exp)
    _check_chunks(data, exp, columns, rg)
    _expected_stats(open(plain, "rb").read(), data)
    assert "GPU SST writer" in pq.ParquetFile(io.BytesIO(data)).metadata.created_by
    # the oracle and the engine read it; aggregates match the oracle's
    assert pa.Table.from_batches(oracle.scan([data], schema.arrow_schema, 2, (), True, 8192).batches).equals(exp)
    assert pa.Table.from_batches(list(eng.scan(handle, [SstInput(id=next(_ids), data=data)], (), None, True))).equals(exp)
    preds = [("tag", "eq", 3)]
    got = eng.scan_aggregate(handle, [SstInput(id=next(_ids), data=data)], preds, group_col=0, ts_col=1, window_ms=60_000, value_col=2)
    want = oracle.scan_aggregate([data], schema.arrow_schema, 2, preds, group_col=0, ts_col=1, window_ms=60_000, value_col=2)
    assert got["series_id"].to_numpy().tolist() == want.gkey.tolist() and got["count"].to_numpy().tolist() == want.count.tolist()
    assert np.array_equal(got["sum"].to_numpy(), want.sum)
    # compacting the encoded output again gives the same rows
    again = str(tmp_path / "again.sst")
    eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=data)], again, max_row_group_size=rg, columns=columns)
    _read_equals(open(again, "rb").read(), exp)
    eng.close()


@pytest.mark.parametrize("rg", [8192, 1000, 97])
@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_encoded_write_batch_matches_the_host_writer(tmp_path, cfg, rg):
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    sid, ts, value, tag = sstgen.synth_columns(0, 12, 250, 1000)
    rng = np.random.default_rng(3)
    perm = rng.permutation(len(sid))                                # write_batch sorts by the primary keys
    batch = pa.RecordBatch.from_arrays([pa.array(sid[perm]), pa.array(ts[perm]), pa.array(value[perm]), pa.array(tag[perm])],
                                       schema=sstgen.METRIC_SCHEMA)
    columns = resolve_column_options(CONFIGS[cfg], schema.arrow_schema)
    eng = Engine(device=0)
    path = str(tmp_path / "w.sst")
    meta = eng.write_batch(handle, batch, 4242, path, max_row_group_size=rg, columns=columns)
    data = open(path, "rb").read()
    assert meta.num_rows == len(sid) and meta.size == len(data)
    want = pq.read_table(io.BytesIO(sstgen.write_sst(schema, batch, 4242, WriteConfig(max_row_group_size=rg, **{
        k: getattr(CONFIGS[cfg], k) for k in ("encoding", "enable_dict", "compression", "column_options")}))))
    _read_equals(data, want)
    _check_chunks(data, want, columns, rg)
    exp = pa.Table.from_batches(oracle.scan([data], schema.arrow_schema, 2, (), True, 8192).batches)
    assert pa.Table.from_batches(list(eng.scan(handle, [SstInput(id=next(_ids), data=data)], (), None, True))).equals(exp)
    eng.close()


def test_page_sizes_against_pyarrow(tmp_path):
    """16 overlapping files of the metric data: uncompressed DELTA data pages of >= 1000 values are no larger than 1.02 x pyarrow's for
    the same values; the index pages of series_id, tag and __seq__ total <= 1.10 x pyarrow's + 64 B per chunk."""
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    datas = [s[0] for s in sstgen.synth_overlapping_ssts(16, series=60, points=1000, delta_ms=1000, keep_frac=0.5, compression="snappy")]
    merged = pa.Table.from_batches(oracle.scan(datas, schema.arrow_schema, 2, (), True, 8192).batches).combine_chunks()
    cfg = WriteConfig(compression="none", column_options={"series_id": ColumnOptions(enable_dict=True), "tag": ColumnOptions(enable_dict=True),
                                                          "__seq__": ColumnOptions(encoding=D), "ts": ColumnOptions(encoding=D)})
    cfg_dict = WriteConfig(compression="none", column_options={n: ColumnOptions(enable_dict=True) for n in ("series_id", "tag", "__seq__")})
    eng = Engine(device=0)
    files = {}
    for key, c in (("delta", cfg), ("dict", cfg_dict)):
        path = str(tmp_path / f"{key}.sst")
        eng.compact_to_sst(handle, _inputs(datas), path, columns=resolve_column_options(c, schema.arrow_schema))
        files[key] = open(path, "rb").read()
        files["pa_" + key] = sstgen.write_sst_with_seq(schema, merged.to_batches()[0], c)
    eng.close()

    def data_pages(data, name):
        md = pq.ParquetFile(io.BytesIO(data)).metadata
        c = md.schema.names.index(name)
        out = []
        for g in range(md.num_row_groups):
            col = md.row_group(g).column(c)
            out.append((col.num_values, sum(len(b) - _levels_end(b) for t, _, b in _chunk_pages(data, col) if t == 0)))
        return out
    for name in ("ts", "__seq__"):
        ours, theirs = data_pages(files["delta"], name), data_pages(files["pa_delta"], name)
        assert len(ours) == len(theirs)
        for (n, a), (_, b) in zip(ours, theirs):
            if n >= 1000:
                assert a <= 1.02 * b, (name, a, b)
    tot_ours = tot_theirs = nchunks = 0
    for name in ("series_id", "tag", "__seq__"):
        ours, theirs = data_pages(files["dict"], name), data_pages(files["pa_dict"], name)
        tot_ours += sum(a for _, a in ours)
        tot_theirs += sum(b for _, b in theirs)
        nchunks += len(ours)
    print(f"\nindex pages: gpu {tot_ours} B, pyarrow {tot_theirs} B over {nchunks} chunks")
    assert tot_ours <= 1.10 * tot_theirs + 64 * nchunks


def _edge_batch():
    rng = np.random.default_rng(8)
    user = arrow_schema([("k", "int64"), ("u8", "uint8"), ("i8", "int8"), ("u16", "uint16"), ("i16", "int16"), ("u32", "uint32"),
                         ("i32", "int32"), ("u64", "uint64"), ("i64", "int64"), ("f32", "float32"), ("f64", "float64"), ("one", "int32")])
    n = 1201
    k = np.arange(n) // 2
    i32 = np.where(np.arange(n) % 2 == 0, -k, 2**31 - 1 - k)                   # deltas 2^31 - 1 and -2^31 in turn: width 32
    u64 = (rng.integers(0, 2**63, n, dtype=np.uint64) | np.uint64(1 << 63)).tolist()       # above 2^63
    i64 = np.where(np.arange(n) % 3 == 0, -2**63, np.where(np.arange(n) % 3 == 1, 2**63 - 1, 0)).tolist()   # min / max side by side: width 64
    nan_payload = np.array([0x7FF8000000000001, 0x7FF0000000000002, 0xFFF8000000000000], dtype=np.uint64).view(np.float64)
    f64 = rng.choice(np.concatenate([nan_payload, [0.0, -0.0, 1.5]]), n).tolist()
    f32 = rng.choice(np.array([np.nan, -0.0, 0.0, 2.5], dtype=np.float32), n).tolist()

    def maybe(vals, p):
        return [None if rng.random() < p else v for v in vals]
    cols = {"k": np.arange(n).tolist(), "u8": maybe(rng.integers(0, 256, n).tolist(), 0.2), "i8": rng.integers(-128, 128, n).tolist(),
            "u16": maybe(rng.integers(0, 65536, n).tolist(), 1.0), "i16": maybe(rng.integers(-32768, 32768, n).tolist(), 0.01),
            "u32": rng.integers(0, 2**32, n).tolist(), "i32": i32.tolist(), "u64": u64, "i64": maybe(i64, 0.1), "f32": f32, "f64": f64,
            "one": [7] * n}
    return user, record_batch(user, cols)


@pytest.mark.parametrize("mode", ["delta", "dict", "dict_delta"])
def test_edge_cases_every_type(tmp_path, mode):
    """Every primitive type; u64 above 2^63, i64 min / max (width 64), alternating i32 min / max (width 32); no, some and all NULLs; NaN
    payloads and +-0.0 (distinct dictionary entries); one distinct value (width 0); a one-row tail chunk; an empty output."""
    user, b = _edge_batch()
    schema = StorageSchema.try_new(user, 1)
    handle = SchemaHandle(schema.arrow_schema, 1)
    ints = [f.name for f in schema.arrow_schema if pa.types.is_integer(f.type)]
    opts = {}
    for f in schema.arrow_schema:
        enc = D if mode != "dict" and f.name in ints else P
        opts[f.name] = ColumnOptions(encoding=enc, enable_dict=mode != "delta", compression=["none", "snappy", "zstd"][len(opts) % 3])
    columns = resolve_column_options(WriteConfig(column_options=opts), schema.arrow_schema)
    assert columns is not None
    data = sstgen.write_sst(schema, b, seq=77, cfg=WriteConfig(max_row_group_size=400))
    exp = pa.Table.from_batches(oracle.scan([data], schema.arrow_schema, 1, (), True, 8192).batches)
    eng = Engine(device=0)
    path = str(tmp_path / "e.sst")
    meta = eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=data)], path, max_row_group_size=600, columns=columns)
    out = open(path, "rb").read()
    assert meta.num_rows == 1201
    md = pq.ParquetFile(io.BytesIO(out)).metadata
    assert md.num_row_groups == 3 and md.row_group(2).num_rows == 1
    _read_equals(out, exp)
    _check_chunks(out, exp, columns, 600)
    again = pa.Table.from_batches(oracle.scan([out], schema.arrow_schema, 1, (), True, 8192).batches)
    assert all(arrays_equal(again[n], exp[n]) for n in exp.schema.names)
    rescan = pa.Table.from_batches(list(eng.scan(handle, [SstInput(id=next(_ids), data=out)], (), None, True)))
    assert all(arrays_equal(rescan[n], exp[n]) for n in exp.schema.names)
    # bit widths at the limits of the physical types
    c32 = exp.schema.names.index("i32")
    if mode == "delta":
        for c, pw, top in ((c32, 4, 32), (exp.schema.names.index("u64"), 8, 64)):
            body = _chunk_pages(out, md.row_group(0).column(c))[0][2]
            assert max(_delta_widths(body[_levels_end(body):], pw)[1]) == top
        one = _chunk_pages(out, md.row_group(0).column(exp.schema.names.index("one")))[0][2]
        assert set(_delta_widths(one[_levels_end(one):], 4)[1]) == {0}
    # an empty output
    empty = sstgen.write_sst(schema, b.slice(0, 0), seq=78)
    path = str(tmp_path / "empty.sst")
    meta = eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=empty)], path, columns=columns)
    assert meta.num_rows == 0 and pq.read_table(path).num_rows == 0
    eng.close()


@pytest.mark.parametrize("fallback", [P, D])
def test_dictionary_over_one_mebibyte_falls_back(tmp_path, fallback):
    """A 200 000-row group with 150 000 distinct 8-byte values: its dictionary page would exceed 1 MiB, so the chunk is written with the
    column's encoding and no dictionary; the small-cardinality column next to it keeps its dictionary."""
    user = arrow_schema([("k", "int64"), ("few", "uint64")])
    schema = StorageSchema.try_new(user, 1)
    handle = SchemaHandle(schema.arrow_schema, 1)
    n = 200_000
    k = (np.arange(n) * 7) % 150_000 + np.arange(n) // 150_000 * 10**9
    b = record_batch(user, {"k": k.tolist(), "few": (np.arange(n) % 5).tolist()})
    columns = resolve_column_options(WriteConfig(enable_dict=True, encoding=fallback, compression="snappy",
                                                 column_options={"few": ColumnOptions(encoding=P)}), schema.arrow_schema)
    eng = Engine(device=0)
    path = str(tmp_path / "big.sst")
    eng.write_batch(handle, b, 9, path, max_row_group_size=n, columns=columns)
    data = open(path, "rb").read()
    md = pq.ParquetFile(io.BytesIO(data)).metadata
    col = md.row_group(0).column(0)
    assert not col.has_dictionary_page
    assert set(col.encodings) == ({"PLAIN", "RLE"} if fallback == P else {"RLE", "DELTA_BINARY_PACKED"})
    assert md.row_group(0).column(1).has_dictionary_page
    want = pa.Table.from_batches([schema.fill_builtin_columns(sstgen.sort_batch(schema, b), 9)])
    _read_equals(data, want)
    got = pa.Table.from_batches(oracle.scan([data], schema.arrow_schema, 1, (), True, 8192).batches)
    assert all(arrays_equal(got[name], want[name]) for name in want.schema.names)
    eng.close()


def test_refused_options_name_the_column(tmp_path):
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    data, _ = sstgen.synth_sst(0, 4, 50, 1000, seq=5)
    eng = Engine(device=0)
    base = [("PLAIN", False, "snappy")] * 6
    for bad, name in (((D, False, "snappy"), "value"), (("PLAIN", False, "gzip"), "tag"), (("RLE", False, "none"), "ts")):
        columns = list(base)
        columns[schema.arrow_schema.names.index(name)] = bad
        for call in (lambda: eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=data)], str(tmp_path / "x.sst"), columns=columns),
                     lambda: eng.write_batch(handle, pa.RecordBatch.from_arrays([pa.array([1], pa.uint64()), pa.array([2], pa.int64()),
                                                                                 pa.array([0.5]), pa.array([1], pa.uint32())],
                                                                                schema=sstgen.METRIC_SCHEMA), 1, str(tmp_path / "y.sst"), columns=columns)):
            with pytest.raises(HgError) as ei:
                call()
            assert ei.value.code == 2 and f"'{name}'" in str(ei.value), str(ei.value)
    buser = arrow_schema([("k", "int64"), ("blob", "binary")])
    bschema = StorageSchema.try_new(buser, 1)
    bh = SchemaHandle(bschema.arrow_schema, 1)
    with pytest.raises(HgError) as ei:
        eng.write_batch(bh, record_batch(buser, {"k": [1], "blob": [b"x"]}), 1, str(tmp_path / "z.sst"), columns=[("PLAIN", False, "none")] * 4)
    assert ei.value.code == 2 and "'blob'" in str(ei.value)
    eng.close()


def test_storage_writes_and_compacts_on_the_gpu(tmp_path, golden):
    """ObjectBasedStorage with dictionary / DELTA options: write and compaction go through the GPU writer; the scans equal those of the
    same batches written by the host writer (pyarrow with the same options)."""
    from horaedb_b200.storage import ObjectBasedStorage, ScanRequest, StorageConfig, WriteRequest
    from horaedb_b200.types import TimeRange, Timestamp
    g = golden["test_storage_write_and_scan"]
    user = arrow_schema(g["schema"])
    eng = Engine(device=0)
    ints = [n for n, t in g["schema"] if "int" in t]
    wcfg = WriteConfig(enable_dict=True, column_options={ints[-1]: ColumnOptions(enable_dict=False, encoding=D, compression="zstd")})
    storage = ObjectBasedStorage(str(tmp_path), g["segment_duration_ms"], user, g["num_primary_keys"], StorageConfig(write=wcfg), engine=eng)
    twins = []
    for w in g["writes"]:
        batch = record_batch(user, w)
        storage.write(WriteRequest(batch, TimeRange(*w["time_range"]), enable_check=True))
        twins.append(sstgen.write_sst(storage.schema_, batch, storage.manifest.ssts[-1].id(), wcfg))
    written = sorted(tmp_path.rglob("*.sst"))
    assert written and all("GPU SST writer" in pq.ParquetFile(p).metadata.created_by for p in written)
    full = TimeRange.new(Timestamp(0), Timestamp.MAX)
    before = pa.Table.from_batches(list(storage.scan(ScanRequest(full, [], None))))
    host = pa.Table.from_batches(oracle.scan(twins, storage.schema_.arrow_schema, g["num_primary_keys"], (), False, 8192).batches)
    assert all(arrays_equal(before[n], host[n]) for n in host.schema.names)
    new = storage.compact()
    assert new
    after_files = set(tmp_path.rglob("*.sst")) - set(written)
    assert after_files and all("RLE_DICTIONARY" in pq.ParquetFile(p).metadata.created_by for p in after_files)
    after = pa.Table.from_batches(list(storage.scan(ScanRequest(full, [], None))))
    assert after.equals(before)
    eng.close()


def test_mixed_output_is_pinned(tmp_path):
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    datas = [s[0] for s in sstgen.synth_overlapping_ssts(3, series=20, points=300, delta_ms=1000, keep_frac=0.5, compression="snappy", seed=11)]
    columns = resolve_column_options(CONFIGS["mixed"], schema.arrow_schema)
    eng = Engine(device=0)
    digests = []
    for i in range(2):
        path = str(tmp_path / f"p{i}.sst")
        eng.compact_to_sst(handle, _inputs(datas), path, max_row_group_size=1000, columns=columns)
        digests.append(hashlib.sha256(open(path, "rb").read()).hexdigest())
    eng.close()
    assert digests[0] == digests[1]
    assert digests[0] == PINNED_SHA256, digests[0]


# SHA-256 of the files of test_every_type_output_is_pinned.  Compaction of the rows and hg_write_batch of the same rows write the same
# bytes; "dict_delta" equals "dict" because every dictionary fits, so DELTA (the fallback) is never used.
EVERY_TYPE_SHA256 = {
    "plain": "9bc524526ac1dd47b06a19b7d64012a4bab3b6f25eca14168961146049f0b354",
    "delta": "57628f0d9c002540ea67250fbf82d3d9b083f997768f166b1b7d941fa22e8bb5",
    "dict": "86210a073a23a94d940e241139a1d750548fcb78c3bc47ff6aa33b2810d7e79e",
    "dict_delta": "86210a073a23a94d940e241139a1d750548fcb78c3bc47ff6aa33b2810d7e79e",
}


@pytest.mark.parametrize("mode", ["plain", "delta", "dict", "dict_delta"])
def test_every_type_output_is_pinned(tmp_path, mode):
    """The bytes of _edge_batch written with every type's statistics (i8 / i16 / i32 / f32, NaN payloads, +-0.0), per-column codecs and
    encodings, and (plain) two bloom filters, through compaction and through hg_write_batch."""
    user, b = _edge_batch()
    schema = StorageSchema.try_new(user, 1)
    handle = SchemaHandle(schema.arrow_schema, 1)
    ints = [f.name for f in schema.arrow_schema if pa.types.is_integer(f.type)]
    opts = {}
    for f in schema.arrow_schema:
        enc = D if mode in ("delta", "dict_delta") and f.name in ints else P
        opts[f.name] = ColumnOptions(encoding=enc, enable_dict=mode.startswith("dict"), compression=["none", "snappy", "zstd"][len(opts) % 3])
    columns = resolve_column_options(WriteConfig(column_options=opts), schema.arrow_schema)
    blooms = [mode == "plain" and f.name in ("i32", "f64") for f in schema.arrow_schema]
    data = sstgen.write_sst(schema, b, seq=77, cfg=WriteConfig(max_row_group_size=400))
    eng = Engine(device=0)
    calls = {"compact": lambda path: eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=data)], path, max_row_group_size=600,
                                                        columns=columns, bloom_filters=blooms, bloom_filter_bytes=4096),
             "write_batch": lambda path: eng.write_batch(handle, b, 77, path, max_row_group_size=600, columns=columns,
                                                         bloom_filters=blooms, bloom_filter_bytes=4096)}
    digests = {}
    for name, call in calls.items():
        for i in range(2):
            path = str(tmp_path / f"{name}{i}.sst")
            call(path)
            digests[(name, i)] = hashlib.sha256(open(path, "rb").read()).hexdigest()
    eng.close()
    assert set(digests.values()) == {EVERY_TYPE_SHA256[mode]}, digests
