"""Binary columns written with a dictionary (`enable_dict`, storage.rs:271-283) or DELTA_BYTE_ARRAY (`ParquetEncoding::DeltaByteArray`,
config.rs:54-75) on the GPU path: scan, merge, dedup, Append concatenation and hg_compact_open.  Oracle as in test_gpu_binary_append.py:
pyarrow decodes the SSTs independently and oracle/merge_stream.py runs MergeStream.  Damaged pages of both encodings end in
HG_ERR_FORMAT (hand-built pages for the rules a random flip rarely hits)."""
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import Engine, HgError, SchemaHandle, SstInput
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode

from helpers import arrays_equal, arrow_schema, record_batch
from test_gpu_binary_append import _check, _reference_scan

pytestmark = pytest.mark.gpu
_ids = iter(range(120_000_000, 124_000_000))
CODECS = [ParquetCompression.Snappy, ParquetCompression.Uncompressed, ParquetCompression.Zstd]
USER = arrow_schema([("pk1", "uint64"), ("pk2", "int32"), ("blob", "binary"), ("idx", "binary")])
HG_ERR_FORMAT = 4


# ------------------------------------------------------------------------------------------------ page headers (thrift compact)
def _varint(b, p):
    r = sh = 0
    while True:
        x = b[p]
        p += 1
        r |= (x & 0x7F) << sh
        sh += 7
        if not x & 0x80:
            return r, p


def _struct(b, p):
    """-> ({field id: int value or nested dict}, end position) for the fields a page header needs."""
    out, fid = {}, 0
    while True:
        h = b[p]
        p += 1
        if h == 0:
            return out, p
        t = h & 0x0F
        fid = fid + (h >> 4) if h >> 4 else None
        if fid is None:
            z, p = _varint(b, p)
            fid = (z >> 1) ^ -(z & 1)
        if t in (1, 2):
            out[fid] = t == 1
        elif t == 3:
            out[fid] = b[p]
            p += 1
        elif t in (4, 5, 6):
            z, p = _varint(b, p)
            out[fid] = (z >> 1) ^ -(z & 1)
        elif t == 8:
            n, p = _varint(b, p)
            p += n
        elif t == 12:
            out[fid], p = _struct(b, p)
        else:
            raise ValueError("unexpected thrift type %d" % t)


def pages(data, rg, col):
    """[(page type, encoding, num_values, payload offset, compressed size)] of one column chunk, dictionary page first."""
    c = pq.ParquetFile(io.BytesIO(data)).metadata.row_group(rg).column(col)
    p = c.dictionary_page_offset if c.has_dictionary_page else c.data_page_offset
    end, out = p + c.total_compressed_size, []
    while p < end:
        h, q = _struct(data, p)
        sub = h.get(5) or h.get(7) or h.get(8) or {}
        enc = sub.get(2) if 8 not in h else sub.get(4)
        out.append((h[1], enc, sub.get(1), q, h[3]))
        p = q + h[3]
    return out


# ----------------------------------------------------------------------------------------------------------------- data
def _rows(rng, nrows, seq, keyspace, f, min_len, kind):
    pk1 = np.sort(rng.integers(0, keyspace, nrows))
    pk2 = rng.integers(-2, 3, nrows)
    order = np.lexsort((pk2, pk1))
    pk1, pk2 = pk1[order], pk2[order]
    keep = np.ones(len(pk1), bool)
    keep[1:] = (pk1[1:] != pk1[:-1]) | (pk2[1:] != pk2[:-1])          # no duplicate PKs inside a file
    pk1, pk2 = pk1[keep], pk2[keep]
    n = len(pk1)
    if kind == "prefix":              # sorted, prefix-sharing values like log lines: DELTA_BYTE_ARRAY's home ground
        blob = [b"host-%05d/cpu/%d/" % (int(k) % 97, int(k) % 3) + b"x" * int(rng.integers(min_len, 9)) for k in pk1]
    elif kind == "low":
        pool = [rng.bytes(int(rng.integers(min_len, 12))) for _ in range(7)]
        blob = [pool[int(rng.integers(0, 7))] for _ in range(n)]
    else:
        blob = [rng.bytes(int(rng.integers(min_len, 40))) for _ in range(n)]
    # a key is NULL in at most one file ((pk1 + f) % 7): a run of several rows never has zero bytes in Append mode
    blob = [None if (int(k) + f) % 7 == 0 else v for k, v in zip(pk1, blob)]
    idx = [b"label-%d" % (seq % 3) if i % 5 else b"" if min_len == 0 else b"z" for i in range(n)]
    return record_batch(USER, {"pk1": pk1.tolist(), "pk2": pk2.tolist(), "blob": blob, "idx": idx})


def _scan_all(eng, handle, schema, datas, append):
    for keep_builtin in (False, True):
        got = list(eng.scan(handle, [SstInput(id=next(_ids), data=d) for d in datas], (), None, keep_builtin))
        _check(got, _reference_scan(schema, datas, append, keep_builtin))


def _encodings(data, col=2):
    md = pq.ParquetFile(io.BytesIO(data)).metadata
    return {e for g in range(md.num_row_groups) for e in md.row_group(g).column(col).encodings}


# ---------------------------------------------------------------------------------------------------------- dictionaries
@pytest.mark.parametrize("codec", CODECS)
def test_dictionary_binary_columns_match_merge_stream(codec):
    rng = np.random.default_rng(61)
    eng = Engine(device=0)
    cfgs = [WriteConfig(compression=codec, max_row_group_size=1000, enable_dict=True),       # numeric columns get dictionaries too
            WriteConfig(compression=codec, max_row_group_size=1000, column_options={"blob": ColumnOptions(enable_dict=True)})]
    for append in (False, True):
        mode = UpdateMode.Append if append else UpdateMode.Overwrite
        schema = StorageSchema.try_new(USER, 2, mode)
        handle = SchemaHandle(schema.arrow_schema, 2, mode)
        ml = 1 if append else 0
        for ci, cfg in enumerate(cfgs):
            kind = ("low", "high")[ci]
            cases = [[_rows(rng, 3000, 5, 400, 0, 0, kind)],                                               # one file, several row groups
                     [_rows(rng, 2500, 10 + f, 300, f, ml, kind) for f in range(4)],                       # overlapping files: a real merge
                     [_rows(rng, 9000, 20 + f, 2000, f, ml, kind) for f in range(3)] + [_rows(rng, 0, 30, 10, 0, 0, kind)]]   # carry; empty
            for batches in cases:
                datas = [sstgen.write_sst(schema, b, seq=100 + i, cfg=cfg, presorted=True) for i, b in enumerate(batches)]
                assert "RLE_DICTIONARY" in _encodings(datas[0])
                _scan_all(eng, handle, schema, datas, append)
    eng.close()


def test_dictionary_fallback_mid_chunk():
    """One row group whose distinct Binary values pass parquet's 1 MiB dictionary page limit: the chunk holds RLE_DICTIONARY pages, then
    PLAIN pages (parquet-rs and pyarrow fall back mid-chunk).  Written with the reference's defaults plus enable_dict."""
    rng = np.random.default_rng(67)
    eng = Engine(device=0)
    n = 8192
    for append in (False, True):
        mode = UpdateMode.Append if append else UpdateMode.Overwrite
        schema = StorageSchema.try_new(USER, 2, mode)
        handle = SchemaHandle(schema.arrow_schema, 2, mode)
        datas = []
        for f in range(2):
            pk1 = np.arange(n, dtype=np.uint64) * 2 + f * 3000
            blob = [None if (int(k) + f) % 11 == 0 else rng.bytes(200) for k in pk1]
            b = record_batch(USER, {"pk1": pk1.tolist(), "pk2": [1] * n, "blob": blob, "idx": [b"ab"] * n})
            datas.append(sstgen.write_sst(schema, b, seq=10 + f, cfg=WriteConfig(enable_dict=True), presorted=True))
        encs = {(t, e) for t, e, _, _, _ in pages(datas[0], 0, 2)}
        assert (2, 0) in encs or (2, 2) in encs                         # the dictionary page
        assert (0, 8) in encs and (0, 0) in encs, encs                  # RLE_DICTIONARY data pages, then PLAIN ones
        _scan_all(eng, handle, schema, datas, append)
        _scan_all(eng, handle, schema, datas[:1], append)
    eng.close()


# ------------------------------------------------------------------------------------------------------- DELTA_BYTE_ARRAY
def _dba_batch(rng, n, seq, f):
    """Sorted prefix-sharing values, repeats (empty suffix), values that extend their predecessor (prefix = the whole previous value),
    empty values, NULL runs, one value over 64 KiB."""
    pk1 = np.arange(n, dtype=np.uint64) * 3 + f
    blob, prev = [], b""
    for i in range(n):
        r = rng.random()
        if (i // 40) % 9 == 4 and (i + f) % 3:                          # NULL runs (some of them start a page)
            blob.append(None)
            continue
        if r < 0.15:
            v = prev                                                    # equal to its predecessor: empty suffix
        elif r < 0.3:
            v = prev + b"/%d" % (i % 10)                               # prefix = the whole previous value
        elif r < 0.35:
            v = b""
        else:
            v = b"host-%05d/cpu/%d/" % (i // 50, i % 4) + rng.bytes(int(rng.integers(0, 20)))
        blob.append(v)
        prev = v
    blob[n // 2] = b"big-" + rng.bytes(70_000)
    idx = [b"region-%d" % ((i // 100) % 3) for i in range(n)]
    return record_batch(USER, {"pk1": pk1.tolist(), "pk2": (pk1 % 5 - 2).astype(np.int32).tolist(), "blob": blob, "idx": idx})


def _write_direct(schema, batch, seq, codec, version, page_size, enc="DELTA_BYTE_ARRAY"):
    """pyarrow directly: small data pages and DataPage V2, which WriteConfig does not reach."""
    full = schema.fill_builtin_columns(batch, seq)
    sink = io.BytesIO()
    pq.write_table(pa.Table.from_batches([full]), sink, row_group_size=1500, compression=codec, use_dictionary=False, data_page_size=page_size, write_batch_size=64,
                   data_page_version=version, column_encoding={"blob": enc, "idx": enc}, write_statistics=True)
    return sink.getvalue()


@pytest.mark.parametrize("codec", CODECS)
def test_delta_byte_array_binary_columns(codec):
    rng = np.random.default_rng(71)
    opts = {"blob": ColumnOptions(encoding=ParquetEncoding.DeltaByteArray), "idx": ColumnOptions(encoding=ParquetEncoding.DeltaByteArray)}
    eng = Engine(device=0)
    for append in (False, True):
        mode = UpdateMode.Append if append else UpdateMode.Overwrite
        schema = StorageSchema.try_new(USER, 2, mode)
        handle = SchemaHandle(schema.arrow_schema, 2, mode)
        batches = [_dba_batch(rng, 3000, 40 + f, f) for f in range(3)]
        via_config = [sstgen.write_sst(schema, b, seq=100 + i, cfg=WriteConfig(compression=codec, max_row_group_size=1000, column_options=opts),
                                       presorted=True) for i, b in enumerate(batches)]
        direct = [_write_direct(schema, b, 200 + i, codec, ver, 2000) for i, (b, ver) in enumerate(zip(batches, ("1.0", "2.0", "2.0")))]
        assert "DELTA_BYTE_ARRAY" in _encodings(via_config[0]) and "DELTA_BYTE_ARRAY" in _encodings(direct[1])
        assert len(pages(direct[1], 0, 2)) > 2                          # several pages per chunk
        for datas in (via_config, direct, via_config[:1], direct[1:2]):
            _scan_all(eng, handle, schema, datas, append)
    eng.close()


# ------------------------------------------------------------------------------------- mixed files, load paths, entry points
def _mixed_files(schema, rng, codec=ParquetCompression.Snappy):
    batches = [_rows(rng, 2500, 60 + f, 600, f, 1, "prefix") for f in range(4)]
    cfgs = [WriteConfig(compression=codec, max_row_group_size=700),
            WriteConfig(compression=codec, max_row_group_size=700, column_options={c: ColumnOptions(encoding=ParquetEncoding.DeltaLengthByteArray) for c in ("blob", "idx")}),
            WriteConfig(compression=codec, max_row_group_size=700, enable_dict=True),
            WriteConfig(compression=codec, max_row_group_size=700, column_options={c: ColumnOptions(encoding=ParquetEncoding.DeltaByteArray) for c in ("blob", "idx")})]
    return [sstgen.write_sst(schema, b, seq=300 + i, cfg=c, presorted=True) for i, (b, c) in enumerate(zip(batches, cfgs))]


def test_mixed_encodings_in_one_call():
    rng = np.random.default_rng(73)
    eng = Engine(device=0)
    for append in (False, True):
        mode = UpdateMode.Append if append else UpdateMode.Overwrite
        schema = StorageSchema.try_new(USER, 2, mode)
        datas = _mixed_files(schema, rng)
        assert {e for t, e, _, _, _ in pages(datas[0], 0, 2) if t == 0} == {0}
        for d, enc in zip(datas[1:], ("DELTA_LENGTH_BYTE_ARRAY", "RLE_DICTIONARY", "DELTA_BYTE_ARRAY")):
            assert enc in _encodings(d)
        _scan_all(eng, SchemaHandle(schema.arrow_schema, 2, mode), schema, datas, append)
    eng.close()


@pytest.mark.parametrize("append", [False, True])
def test_resident_transient_predicates_and_compaction(append):
    rng = np.random.default_rng(79)
    mode = UpdateMode.Append if append else UpdateMode.Overwrite
    schema = StorageSchema.try_new(USER, 2, mode)
    handle = SchemaHandle(schema.arrow_schema, 2, mode)
    datas = _mixed_files(schema, rng, ParquetCompression.Zstd)
    eng = Engine(device=0)
    ids = [next(_ids) for _ in datas]
    for i, d in zip(ids, datas):
        eng.load_sst(handle, SstInput(id=i, data=d))
    for keep_builtin in (False, True):
        exp = _reference_scan(schema, datas, append, keep_builtin)
        _check(list(eng.scan(handle, [SstInput(id=i) for i in ids], (), None, keep_builtin)), exp)                          # resident
        _check(list(eng.scan(handle, [SstInput(id=next(_ids), data=d) for d in datas], (), None, keep_builtin)), exp)      # transient
    # hg_compact_open = the merged stream with the builtin columns
    _check(list(eng.compact(handle, [SstInput(id=i) for i in ids])), _reference_scan(schema, datas, append, True))
    _check(list(eng.compact(handle, [SstInput(id=next(_ids), data=d) for d in datas])), _reference_scan(schema, datas, append, True))
    # a predicate on a fixed-width column in front of the merge: same as scanning pre-filtered files
    for ins in ([SstInput(id=i) for i in ids], [SstInput(id=next(_ids), data=d) for d in datas]):
        got = pa.Table.from_batches(list(eng.scan(handle, ins, [("pk2", "ge", 0)], None, False)), schema=schema.user_schema())
        filt = []
        for d in datas:
            t = pq.read_table(io.BytesIO(d))
            t = t.filter(pa.compute.greater_equal(t["pk2"], 0)).combine_chunks()
            filt.append(sstgen.write_sst_with_seq(schema, t.to_batches()[0], WriteConfig(max_row_group_size=1000)))
        exp_tbl = pa.Table.from_batches(_reference_scan(schema, filt, append, False), schema=schema.user_schema())
        assert got.num_rows == exp_tbl.num_rows > 0
        for name in exp_tbl.schema.names:
            assert arrays_equal(got[name], exp_tbl[name]), name
    for i in ids:
        eng.unload_sst(i)
    eng.close()


def test_device_to_host_traffic_only_for_delta_byte_array():
    """A dictionary call copies and launches exactly what the PLAIN call does; a DELTA_BYTE_ARRAY call adds one small copy of the page
    sizes and one kernel (dba_materialise)."""
    rng = np.random.default_rng(83)
    schema = StorageSchema.try_new(USER, 2)
    handle = SchemaHandle(schema.arrow_schema, 2)
    b = _rows(rng, 4000, 5, 100_000, 0, 0, "prefix")
    opts = {c: ColumnOptions(encoding=ParquetEncoding.DeltaByteArray) for c in ("blob", "idx")}
    plain, dic, dba = (sstgen.write_sst(schema, b, seq=9, cfg=c, presorted=True)
                       for c in (WriteConfig(max_row_group_size=1000), WriteConfig(max_row_group_size=1000, column_options={"blob": ColumnOptions(enable_dict=True), "idx": ColumnOptions(enable_dict=True)}),
                                 WriteConfig(max_row_group_size=1000, column_options=opts)))
    eng = Engine(device=0)
    got, st = {}, {}
    for name, d in (("plain", plain), ("dict", dic), ("dba", dba)):
        got[name] = pa.Table.from_batches(list(eng.scan(handle, [SstInput(id=next(_ids), data=d)])))
        st[name] = eng.stats()
    assert got["plain"].equals(got["dict"]) and got["plain"].equals(got["dba"])
    assert st["dict"]["bytes_d2h"] == st["plain"]["bytes_d2h"] and st["dict"]["kernel_launches"] == st["plain"]["kernel_launches"]
    assert st["dba"]["bytes_d2h"] > st["plain"]["bytes_d2h"] and st["dba"]["kernel_launches"] == st["plain"]["kernel_launches"] + 1
    eng.close()


# ------------------------------------------------------------------------------------------------------- hand-built damage
def _one_page_sst(values, enc, seq=1):
    """One uncompressed V1 page per Binary chunk, no NULLs: -> (schema, handle, bytes, payload offset of the blob page)."""
    schema = StorageSchema.try_new(USER, 2)
    n = len(values)
    b = record_batch(USER, {"pk1": list(range(n)), "pk2": [0] * n, "blob": values, "idx": [b"i"] * n})
    full = schema.fill_builtin_columns(b, seq)
    sink = io.BytesIO()
    kw = dict(use_dictionary=["blob"]) if enc == "dict" else dict(use_dictionary=False, column_encoding={"blob": enc})
    pq.write_table(pa.Table.from_batches([full]), sink, compression="none", data_page_version="1.0", **kw)
    data = sink.getvalue()
    pg = [p for p in pages(data, 0, 2) if p[0] == 0]
    assert len(pg) == 1
    return schema, SchemaHandle(schema.arrow_schema, 2), bytearray(data), pg[0][3]


def _values_at(data, off):
    """Offset of the values section of a V1 page of an optional column: behind [u32 length][definition levels]."""
    return off + 4 + int.from_bytes(data[off:off + 4], "little")


def _expect_format_error(eng, handle, data):
    with pytest.raises(HgError) as ei:
        list(eng.scan(handle, [SstInput(id=next(_ids), data=bytes(data))]))
    assert ei.value.code == HG_ERR_FORMAT, str(ei.value)


def test_hand_built_damage_is_a_format_error():
    eng = Engine(device=0)
    # DELTA_BYTE_ARRAY over 1-byte values with nothing in common: prefix run = [128][4][n][first 0][min delta 0][4 bit widths 0]
    vals = [bytes([97 + i % 3]) for i in range(20)]
    schema, handle, data, off = _one_page_sst(vals, "DELTA_BYTE_ARRAY")
    _check(list(eng.scan(handle, [SstInput(id=next(_ids), data=bytes(data))])), _reference_scan(schema, [bytes(data)], False, False))
    v = _values_at(data, off)
    assert data[v:v + 5] == bytes([0x80, 0x01, 0x04, 20, 0x00]) and data[v + 5] == 0x00        # prefix run: first 0, min delta 0
    s = v + 10                                                                                  # suffix run: first 1 (zigzag 2)
    assert data[s:s + 5] == bytes([0x80, 0x01, 0x04, 20, 0x02])
    bad = bytearray(data); bad[v + 4] = 0x02                                                   # prefix[0] = 1
    _expect_format_error(eng, handle, bad)
    bad = bytearray(data); bad[v + 5] = 0x04                                                   # prefix[i] = 2i > length of value i-1
    _expect_format_error(eng, handle, bad)
    bad = bytearray(data); bad[s + 4] = 0x7E                                                   # 63-byte suffixes: past the page
    _expect_format_error(eng, handle, bad)
    # dictionary of 3 entries (bit width 2): one bit-packed group of indices set to 3 = the entry count
    schema, handle, data, off = _one_page_sst([b"aa", b"b", b"cccc"] * 8, "dict")
    _check(list(eng.scan(handle, [SstInput(id=next(_ids), data=bytes(data))])), _reference_scan(schema, [bytes(data)], False, False))
    v = _values_at(data, off)
    assert data[v] == 2 and data[v + 1] & 1                                                    # bit width 2, a bit-packed run
    bad = bytearray(data); bad[v + 2] = 0xFF
    _expect_format_error(eng, handle, bad)
    eng.close()
