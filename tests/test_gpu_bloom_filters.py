"""Split-block bloom filters on the GPU: written by the SST writer (csrc/sst_writer.cu bloom_build_kernel, hg_column_write_opts.bloom_filter)
and used by the scan planner to prune row groups for `=` / `IN` predicates (csrc/engine.cu bloom_prune_resident and rg_survives, the host
test of transient loads and hg_plan_row_groups, csrc/fused_scan.cu prune_rgs_kernel).

The writer's bitsets must equal pyarrow's for the same rows and row-group size (and tests/bloom_model.py's at any size); the reader must
return the oracle's rows, and decode exactly the row groups that statistics plus the model keep — or statistics alone with
HG_FLAG_NO_BLOOM_FILTER."""
import hashlib
import io
import os
import tempfile

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import bloom_model as M
from horaedb_b200 import _ffi, sstgen
from horaedb_b200._ffi import Engine, HgError, SchemaHandle, SstInput
from horaedb_b200.config import ColumnOptions, ParquetEncoding, StorageConfig, WriteConfig, resolve_bloom_filters, resolve_column_options
from horaedb_b200.types import StorageSchema
from oracle import oracle

from helpers import arrays_equal, arrow_schema, record_batch

pytestmark = pytest.mark.gpu
_ids = iter(range(97_000_000, 98_000_000))
D, P = ParquetEncoding.DeltaBinaryPacked, ParquetEncoding.Plain

# SHA-256 of the file of test_output_is_pinned (same rows and options -> same bytes, on the GPU and emulated)
PINNED_SHA256 = "7f8c540ab85107a1318f0ef759dec8dd128c68db8b47b88e4c6ffc8ce02a6dab"

EDGE = arrow_schema([("k", "uint64"), ("u8", "uint8"), ("i8", "int8"), ("u16", "uint16"), ("i16", "int16"), ("u32", "uint32"), ("i32", "int32"),
                     ("i64", "int64"), ("f32", "float32"), ("f64", "float64"), ("nul", "int32")])


def _edge_batch(n=1201, seed=5):
    rng = np.random.default_rng(seed)
    cols = {"k": np.arange(n).tolist()}
    for f in EDGE:
        if f.name in ("k", "nul"):
            continue
        if pa.types.is_floating(f.type):
            v = rng.standard_normal(n).astype(f.type.to_pandas_dtype())
            v[:5] = [np.nan, -0.0, 0.0, np.inf, -np.inf]
            v[5] = np.array([0x7ff8000000000abc], np.uint64).view(np.float64)[0] if f.type == pa.float64() else np.array([0x7fc00abc], np.uint32).view(np.float32)[0]
        else:
            info = np.iinfo(f.type.to_pandas_dtype())
            v = rng.integers(info.min, info.max, n, dtype=f.type.to_pandas_dtype(), endpoint=True)
        vals = v.tolist()
        for i in rng.choice(n, n // 10, replace=False):
            vals[i] = None
        cols[f.name] = vals
    cols["nul"] = [None] * n
    return record_batch(EDGE, cols)


def _bitsets(data):
    """{(row group, column): bitset} of a file, read with the model's own footer walk."""
    out = {}
    for (g, c), ent in M.footer_blooms(data).items():
        if ent["offset"] >= 0:
            nb, hlen, bits = M.read_filter(data, ent["offset"])
            assert ent["length"] == hlen + nb
            out[(g, c)] = bits
    return out


def _read_equals(data, exp):
    got = pq.read_table(io.BytesIO(data))
    assert got.schema.names == exp.schema.names
    for name in exp.schema.names:
        assert arrays_equal(got[name], exp[name]), name


# ------------------------------------------------------------------------------------------------------------------------ writer
MODES = {8192: ("none", "plain"), 1000: ("snappy", "delta"), 97: ("zstd", "dict")}


@pytest.mark.parametrize("rg,nbytes", [(8192, 0), (1000, 0), (97, 4096)])
def test_bitsets_equal_pyarrow(tmp_path, rg, nbytes):
    """Every primitive type (NaN payloads, +-0.0, NULLs, an all-NULL column), PLAIN / DELTA / dictionary chunks, every codec: the
    GPU's filters equal pyarrow's for the same rows, and every reader reads the file."""
    schema = StorageSchema.try_new(EDGE, 1)
    handle = SchemaHandle(schema.arrow_schema, 1)
    codec, mode = MODES[rg]
    ints = [f.name for f in schema.arrow_schema if pa.types.is_integer(f.type)]
    opts = {f.name: ColumnOptions(encoding=D if mode == "delta" and f.name in ints else P, enable_dict=mode == "dict", compression=codec)
            for f in schema.arrow_schema}
    cfg = WriteConfig(enable_bloom_filter=True, column_options=opts, max_row_group_size=rg)
    columns, blooms = resolve_column_options(cfg, schema.arrow_schema), resolve_bloom_filters(cfg, schema.arrow_schema)
    batch = _edge_batch()
    eng = Engine(device=0)
    path = str(tmp_path / "b.sst")
    meta = eng.write_batch(handle, batch, 31, path, max_row_group_size=rg, columns=columns, bloom_filters=blooms, bloom_filter_bytes=nbytes)
    data = open(path, "rb").read()
    assert meta.size == len(data)
    want = pa.Table.from_batches([schema.fill_builtin_columns(sstgen.sort_batch(schema, batch), 31)])
    _read_equals(data, want)
    # pyarrow writes the same rows with the same row groups; an ndv that gives the same bitset size
    sink = io.BytesIO()
    ndv = 1_000_000 if nbytes == 0 else nbytes
    pq.write_table(want, sink, row_group_size=rg, bloom_filter_options={n: {"ndv": ndv, "fpp": 0.05} for n in want.column_names})
    ours, theirs = _bitsets(data), _bitsets(sink.getvalue())
    size = nbytes or (1 << 20)
    assert set(ours) == set(theirs) and len(ours) == pq.ParquetFile(io.BytesIO(data)).metadata.num_row_groups * len(want.column_names)
    for key in ours:
        assert len(theirs[key]) == size and ours[key] == theirs[key], key
        g, c = key
        assert ours[key] == M.build(M.phys_values(want.column(c).slice(g * rg, rg)), size)
    assert "bloom filters" in pq.ParquetFile(io.BytesIO(data)).metadata.created_by
    exp = pa.Table.from_batches(oracle.scan([data], schema.arrow_schema, 1, (), True, 8192).batches)
    assert all(arrays_equal(exp[n], want[n]) for n in want.column_names)
    got = pa.Table.from_batches(list(eng.scan(handle, [SstInput(id=next(_ids), data=data)], (), None, True)))
    assert all(arrays_equal(got[n], want[n]) for n in want.column_names)
    eng.close()


def test_sizes_layout_and_refusals(tmp_path):
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    datas = [s[0] for s in sstgen.synth_overlapping_ssts(3, series=16, points=200, delta_ms=1000, keep_frac=0.5, compression="snappy", seed=3)]
    merged = pa.Table.from_batches(oracle.scan(datas, schema.arrow_schema, 2, (), True, 8192).batches)
    eng = Engine(device=0)
    names = schema.arrow_schema.names
    flags = [n in ("value", "tag") for n in names]
    plain = str(tmp_path / "plain.sst")
    eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=d) for d in datas], plain, max_row_group_size=1000)
    plain_b = open(plain, "rb").read()
    for nbytes in (32, 1024, 65536, 256 << 10):                  # shared-memory bitsets (<= 128 KiB) and global ones
        path = str(tmp_path / f"s{nbytes}.sst")
        eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=d) for d in datas], path, max_row_group_size=1000, bloom_filters=flags,
                           bloom_filter_bytes=nbytes)
        data = open(path, "rb").read()
        _read_equals(data, merged)
        md = pq.ParquetFile(io.BytesIO(data)).metadata
        walk = M.footer_blooms(data)
        pmd = pq.ParquetFile(io.BytesIO(plain_b)).metadata
        for g in range(md.num_row_groups):
            rg = md.row_group(g)
            end = max(rg.column(c).data_page_offset + rg.column(c).total_compressed_size for c in range(len(names)))
            # the filters follow the row group's chunks in column order; chunk sizes are those of the file without filters
            at = end
            for c, n in enumerate(names):
                assert rg.column(c).total_compressed_size == pmd.row_group(g).column(c).total_compressed_size
                ent = walk[(g, c)]
                if not flags[c]:
                    assert ent["offset"] == -1 and ent["length"] == -1
                    continue
                assert ent["offset"] == at
                hdr = data[at:at + ent["length"] - nbytes]
                assert hdr[0] == 0x15 and hdr[-13:] == bytes([0x1c, 0x1c, 0, 0, 0x1c, 0x1c, 0, 0, 0x1c, 0x1c, 0, 0, 0])
                at += ent["length"]
                bits = M.read_filter(data, ent["offset"])[2]
                assert bits == M.build(M.phys_values(merged.column(c).slice(g * 1000, 1000)), nbytes), (nbytes, g, n)
                info = _ffi.parquet_bloom_info(data, g, c)
                assert info["usable"] == 1 and info["num_bytes"] == nbytes
    # all-zero flags write the bytes of no flags at all
    zero = str(tmp_path / "zero.sst")
    eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=d) for d in datas], zero, max_row_group_size=1000, bloom_filters=[False] * len(names))
    assert open(zero, "rb").read() == plain_b
    assert "bloom" not in pq.ParquetFile(io.BytesIO(plain_b)).metadata.created_by
    # refused values, before any device work
    for bad in (16, 48, 100, 3 << 20, 256 << 20):
        with pytest.raises(HgError) as ei:
            eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=d) for d in datas], str(tmp_path / "x.sst"), bloom_filters=flags,
                               bloom_filter_bytes=bad)
        assert ei.value.code == 1 and "bloom_filter_bytes" in str(ei.value)
    with pytest.raises(HgError) as ei:
        eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=d) for d in datas], str(tmp_path / "x.sst"),
                           bloom_filters=[0, 0, 2, 0, 0, 0])
    assert ei.value.code == 2 and "'value'" in str(ei.value)
    eng.close()


def test_storage_writes_and_compacts_with_filters(tmp_path):
    """ObjectBasedStorage with the table-wide flag and a per-column override: write_batch and compaction on the GPU carry filters on
    exactly the resolved columns."""
    from horaedb_b200.storage import ObjectBasedStorage, ScanRequest, WriteRequest
    from horaedb_b200.types import TimeRange, Timestamp
    user = arrow_schema([("host", "uint32"), ("ts", "int64"), ("rid", "uint64"), ("v", "float64")])
    cfg = WriteConfig(enable_bloom_filter=True, max_row_group_size=64, column_options={"ts": ColumnOptions(enable_bloom_filter=False),
                                                                                       "__seq__": ColumnOptions(enable_bloom_filter=False)})
    eng = Engine(device=0)
    st = ObjectBasedStorage(str(tmp_path), 1 << 40, user, 2, StorageConfig(write=cfg), engine=eng)
    rng = np.random.default_rng(2)
    for w in range(5):
        n = 150
        st.write(WriteRequest(record_batch(user, {"host": rng.integers(0, 5, n).tolist(), "ts": rng.integers(0, 1000, n).tolist(),
                                                  "rid": rng.integers(0, 2**63, n).tolist(), "v": rng.standard_normal(n).tolist()}),
                              TimeRange(0, 1000)))
    want = [n not in ("ts", "__seq__") for n in st.schema_.arrow_schema.names]
    files = sorted(tmp_path.rglob("*.sst"))
    written = [open(p, "rb").read() for p in files]
    full = TimeRange.new(Timestamp(0), Timestamp.MAX)
    before = pa.Table.from_batches(list(st.scan(ScanRequest(full, [], None))))
    assert st.compact()
    after_files = sorted(set(tmp_path.rglob("*.sst")) - set(files))
    assert after_files
    for data in written + [open(p, "rb").read() for p in after_files]:
        walk = M.footer_blooms(data)
        assert "GPU SST writer" in pq.ParquetFile(io.BytesIO(data)).metadata.created_by
        assert all((walk[(g, c)]["offset"] >= 0) == want[c] for (g, c) in walk)
    after = pa.Table.from_batches(list(st.scan(ScanRequest(full, [], None))))
    assert after.equals(before)
    eng.close()


def test_output_is_pinned(tmp_path):
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    datas = [s[0] for s in sstgen.synth_overlapping_ssts(3, series=20, points=300, delta_ms=1000, keep_frac=0.5, compression="snappy", seed=11)]
    cfg = WriteConfig(column_options={"series_id": ColumnOptions(enable_dict=True, enable_bloom_filter=True, compression="zstd"),
                                      "ts": ColumnOptions(encoding=D), "value": ColumnOptions(enable_bloom_filter=True),
                                      "tag": ColumnOptions(enable_bloom_filter=True, compression="none")})
    eng = Engine(device=0)
    digests = []
    for i, nbytes in enumerate((2048, 2048)):
        path = str(tmp_path / f"p{i}.sst")
        eng.compact_to_sst(handle, [SstInput(id=next(_ids), data=d) for d in datas], path, max_row_group_size=1000,
                           columns=resolve_column_options(cfg, schema.arrow_schema), bloom_filters=resolve_bloom_filters(cfg, schema.arrow_schema),
                           bloom_filter_bytes=nbytes)
        digests.append(hashlib.sha256(open(path, "rb").read()).hexdigest())
    eng.close()
    assert digests[0] == digests[1]
    assert digests[0] == PINNED_SHA256, digests[0]


# ------------------------------------------------------------------------------------------------------------------------ reader
EVENTS = arrow_schema([("host", "uint64"), ("ts", "int64"), ("rid", "uint64"), ("code", "int32"), ("val", "float64"), ("f32", "float32")])
RG = 250


def _event_files(source, nulls):
    """Two PK-disjoint SSTs sorted by (host, ts) with a random unique rid; filters on rid, code, val and f32 (written by the GPU or by
    pyarrow), and the same rows without filters."""
    rng = np.random.default_rng(7)
    st = StorageSchema.try_new(EVENTS, 2)
    handle = SchemaHandle(st.arrow_schema, 2)
    out = []
    rids = rng.permutation(np.arange(1, 4001, dtype=np.uint64)) * np.uint64(7919)
    for f in range(2):
        n = 2000
        val = rng.integers(-50, 50, n) / 4.0
        val[3], val[4] = -0.0, 0.0
        cols = {"host": (np.arange(n) // 100 + f * 1000).tolist(), "ts": (np.arange(n) % 100 * 1000).tolist(), "rid": rids[f * n:(f + 1) * n].tolist(),
                "code": rng.integers(0, 40, n).tolist(), "val": val.tolist(), "f32": (val * 2).astype(np.float32).tolist()}
        if nulls:                                        # (NULLs also keep the transient late-materialisation gate off)
            for c in ("rid", "code", "val", "f32"):
                for i in range(5, n, 97):
                    cols[c][i] = None
        batch = record_batch(EVENTS, cols)
        bloom = {c: ColumnOptions(enable_bloom_filter=True) for c in ("rid", "code", "val", "f32")}
        without = sstgen.write_sst(st, batch, 10 + f, WriteConfig(max_row_group_size=RG))
        if source == "pyarrow":
            with_f = sstgen.write_sst(st, batch, 10 + f, WriteConfig(max_row_group_size=RG, column_options=bloom))
        else:
            eng = Engine(device=0)
            cfg = WriteConfig(max_row_group_size=RG, column_options=bloom)
            with tempfile.TemporaryDirectory() as tmp:
                path = os.path.join(tmp, "f.sst")
                eng.write_batch(handle, batch, 10 + f, path, max_row_group_size=RG, compression="snappy",
                                bloom_filters=resolve_bloom_filters(cfg, st.arrow_schema), bloom_filter_bytes=4096)
                with_f = open(path, "rb").read()
            eng.close()
        out.append((with_f, without))
    return st, handle, out


def _rows_kept(handle, data, preds):
    keep = _ffi.plan_row_groups(handle, data, preds)
    md = pq.ParquetFile(io.BytesIO(data)).metadata
    return sum(md.row_group(g).num_rows for g, k in enumerate(keep) if k)


def _model_rows(st, handle, with_f, without, preds):
    """Rows of the row groups statistics (hg_plan_row_groups on the file without filters) and the model keep."""
    stats = _ffi.plan_row_groups(handle, without, preds)
    walk = M.footer_blooms(with_f)
    md = pq.ParquetFile(io.BytesIO(with_f)).metadata
    total = 0
    for g, k in enumerate(stats):
        for col, op, lit in preds:
            c = st.arrow_schema.names.index(col)
            ent = walk.get((g, c), {"offset": -1})
            if k and ent["offset"] >= 0 and not M.bloom_keeps(M.read_filter(with_f, ent["offset"])[2], st.arrow_schema.field(c).type, op, lit):
                k = 0
        total += md.row_group(g).num_rows if k else 0
    return total


SCAN_PREDS = [
    [("rid", "eq", 7919 * 123)],
    [("rid", "eq", 7919 * 123 + 1)],
    [("rid", "in", [7919 * 5, 7919 * 3999, 7919 * 77 + 3, 11, 7919 * 2500, 7919 * 10, 7919 * 11, 7919 * 12])],
    [("rid", "eq", 7919 * 321), ("code", "eq", 3)],
    [("rid", "in", [7919 * 321, 7919 * 322]), ("code", "in", [3, 4])],
    [("val", "eq", -0.0)], [("val", "eq", 0.0)], [("val", "eq", float("nan"))], [("val", "eq", 1.25)],
    [("f32", "eq", 2.5)], [("f32", "eq", 0.1)],
    [("rid", "ne", 7919 * 123)],
]


@pytest.mark.parametrize("resident", [True, False])
@pytest.mark.parametrize("source", ["gpu", "pyarrow"])
def test_scan_pruning(source, resident):
    st, handle, files = _event_files(source, nulls=True)
    datas = [w for w, _ in files]
    eng = Engine(device=0)
    ids = [next(_ids) for _ in datas]
    if resident:
        for i, d in zip(ids, datas):
            eng.load_sst(handle, SstInput(id=i, data=d))
    ssts = [SstInput(id=i, data=None if resident else d) for i, d in zip(ids, datas)]
    for preds in SCAN_PREDS:
        want_b = oracle.scan(datas, st.arrow_schema, 2, preds, False, 8192).batches
        want = pa.Table.from_batches(want_b) if want_b else None
        for flags in (0, _ffi.HG_FLAG_NO_FUSED, _ffi.HG_FLAG_NO_BLOOM_FILTER):
            eng.set_flags(flags)
            got_b = list(eng.scan(handle, ssts, preds, None, False))
            if want is None:
                assert sum(b.num_rows for b in got_b) == 0, (preds, flags)
            else:
                got = pa.Table.from_batches(got_b)
                assert got.num_rows == want.num_rows and all(arrays_equal(got[n], want[n]) for n in want.column_names), (preds, flags)
            s = eng.stats()
            if flags & _ffi.HG_FLAG_NO_BLOOM_FILTER:
                assert s["rows_decoded"] == sum(_rows_kept(handle, wo, preds) for _, wo in files), preds
            else:
                assert s["rows_decoded"] == sum(_model_rows(st, handle, w, wo, preds) for w, wo in files), (preds, flags)
                assert s["rows_decoded"] == sum(_rows_kept(handle, w, preds) for w, _ in files)
    # the point lookup decodes one row group instead of all of them
    eng.set_flags(0)
    list(eng.scan(handle, ssts, [("rid", "eq", 7919 * 123)], None, False))
    assert eng.stats()["rows_decoded"] == RG
    eng.close()


@pytest.mark.parametrize("resident", [True, False])
@pytest.mark.parametrize("source", ["gpu", "pyarrow"])
def test_aggregate_pruning_fused_and_general(source, resident):
    st, handle, files = _event_files(source, nulls=False)
    datas = [w for w, _ in files]
    eng = Engine(device=0)
    ids = [next(_ids) for _ in datas]
    if resident:
        for i, d in zip(ids, datas):
            eng.load_sst(handle, SstInput(id=i, data=d))
    ssts = [SstInput(id=i, data=None if resident else d) for i, d in zip(ids, datas)]
    nolm = _ffi.HG_FLAG_NO_LATE_MATERIALIZATION          # transient loads: the gate would prune row groups of its own
    for preds in ([("rid", "eq", 7919 * 123)], [("rid", "eq", 7919 * 123 + 1)], [("rid", "eq", 7919 * 321), ("code", "eq", 3)],
                  [("code", "eq", 41)], [("rid", "in", [7919 * 321, 7919 * 2222])]):
        want = oracle.scan_aggregate(datas, st.arrow_schema, 2, preds, group_col=0, ts_col=1, window_ms=10_000, value_col=4)
        for flags in (nolm, nolm | _ffi.HG_FLAG_NO_FUSED, nolm | _ffi.HG_FLAG_NO_BLOOM_FILTER):
            eng.set_flags(flags)
            got = eng.scan_aggregate(handle, ssts, preds, group_col=0, ts_col=1, window_ms=10_000, value_col=4)
            assert got["host"].to_numpy().tolist() == want.gkey.tolist() and got["count"].to_numpy().tolist() == want.count.tolist(), (preds, flags)
            assert np.array_equal(got["sum"].to_numpy(), want.sum)
            s = eng.stats()
            if all(op == "eq" for _, op, _ in preds) and len(want.gkey) and not flags & _ffi.HG_FLAG_NO_FUSED:
                assert s["path"] & 1, (preds, flags)                 # `=` on integer columns: the fused path
            if flags & _ffi.HG_FLAG_NO_BLOOM_FILTER:
                assert s["rows_decoded"] == sum(_rows_kept(handle, wo, preds) for _, wo in files)
            else:
                assert s["rows_decoded"] == sum(_model_rows(st, handle, w, wo, preds) for w, wo in files), (preds, flags)
    eng.close()


def test_files_without_filters_launch_the_same_kernels():
    st, handle, files = _event_files("pyarrow", nulls=True)
    without = [wo for _, wo in files]
    eng = Engine(device=0)
    ids = [next(_ids) for _ in without]
    for i, d in zip(ids, without):
        eng.load_sst(handle, SstInput(id=i, data=d))
    for resident in (True, False):
        ssts = [SstInput(id=i if resident else next(_ids), data=None if resident else d) for i, d in zip(ids, without)]
        for preds in ([("rid", "eq", 7919 * 123)], [("rid", "in", [7919, 7919 * 2])]):
            launches = []
            for flags in (_ffi.HG_FLAG_NO_FUSED, _ffi.HG_FLAG_NO_FUSED | _ffi.HG_FLAG_NO_BLOOM_FILTER):
                eng.set_flags(flags)
                list(eng.scan(handle, ssts, preds, None, False))
                launches.append(eng.stats()["kernel_launches"])
            assert launches[0] == launches[1], (resident, preds, launches)
    eng.close()


def test_general_pipeline_probes_the_filters_once():
    """The general pipeline selects the row groups of a call once: over resident files with filters, the bloom probe adds exactly one
    launch, for PK-disjoint inputs and for overlapping ones (the same rows under two ids), which are merged and need __seq__."""
    st, handle, files = _event_files("pyarrow", nulls=True)
    datas = [w for w, _ in files]
    rids = [pq.read_table(io.BytesIO(d))["rid"][0].as_py() for d in datas]   # one rid of each file: some row group survives in every file
    eng = Engine(device=0)
    for inputs in (datas, [datas[0], datas[0]]):
        ids = [next(_ids) for _ in inputs]
        for i, d in zip(ids, inputs):
            eng.load_sst(handle, SstInput(id=i, data=d))
        ssts = [SstInput(id=i) for i in ids]
        launches = []
        for flags in (_ffi.HG_FLAG_NO_FUSED, _ffi.HG_FLAG_NO_FUSED | _ffi.HG_FLAG_NO_BLOOM_FILTER):
            eng.set_flags(flags)
            list(eng.scan(handle, ssts, [("rid", "in", rids)], None, False))
            launches.append(eng.stats()["kernel_launches"])
            if not flags & _ffi.HG_FLAG_NO_BLOOM_FILTER:
                assert eng.stats()["rows_decoded"] == 2 * RG
        assert launches[0] == launches[1] + 1, (inputs is datas, launches)
    eng.close()
