"""Gate bits of the fused scan (fused_scan.cu): on a gate-first Snappy call, the row-group gate kernel keeps one bit per row of the gate
column and the fused kernel's gate sweeps read the bits instead of the values.  Every case is checked against the oracle (f64 sums bit-exact) and against the
same call under HG_FLAG_NO_LATE_MATERIALIZATION, which has no gate-first job and so no bits."""
import numpy as np
import pyarrow as pa
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import HG_FLAG_NO_LATE_MATERIALIZATION, Engine, SchemaHandle, SstInput
from horaedb_b200.config import ParquetCompression, WriteConfig
from horaedb_b200.types import StorageSchema
from oracle import oracle

pytestmark = pytest.mark.gpu
_ids = iter(range(70_000_000, 80_000_000))
SNAPPY, NONE = ParquetCompression.Snappy, ParquetCompression.Uncompressed


def _schema(gate_type, nullable=True):
    fields = [pa.field("series_id", pa.uint64(), nullable), pa.field("ts", pa.int64(), nullable), pa.field("value", pa.float64(), nullable),
              pa.field("tag", gate_type, nullable)]
    schema = StorageSchema.try_new(pa.schema(fields), 2)
    schema.user_arrow = pa.schema(fields)
    return schema


def _write(schema, sid, ts, value, tag, rg, compression, seq):
    arrow = schema.user_arrow
    batch = pa.RecordBatch.from_arrays([pa.array(sid.astype(np.uint64)), pa.array(ts.astype(np.int64)), pa.array(value.astype(np.float64)),
                                        pa.array(tag, type=arrow.field("tag").type)], schema=arrow)
    return sstgen.write_sst(schema, batch, seq=seq, cfg=WriteConfig(compression=compression, max_row_group_size=rg), presorted=True)


def _rows(n, nseries, lo, rng):
    sid = np.sort(rng.integers(lo, lo + nseries, n))
    ts = sstgen.T0_MS + np.arange(n) * 1000
    return sid, ts, rng.random(n) * 100 - 50


def _check(got, exp, bucket):
    assert got.num_rows == len(exp.count)
    if got.num_rows:
        assert got["series_id"].to_numpy().tolist() == exp.gkey.tolist()
        if bucket:
            assert got["bucket"].to_numpy().tolist() == exp.bucket.tolist()
        assert got["count"].to_numpy().tolist() == exp.count.tolist()
        assert np.array_equal(got["sum"].to_numpy(), exp.sum) and np.array_equal(got["min"].to_numpy(), exp.min)
        assert np.array_equal(got["max"].to_numpy(), exp.max)


def _run(schema, datas, preds, kw, fused=True):
    handle = SchemaHandle(schema.arrow_schema, 2)
    exp = oracle.scan_aggregate(datas, schema.arrow_schema, 2, preds, **kw)
    res = []
    for flags in (0, HG_FLAG_NO_LATE_MATERIALIZATION):
        eng = Engine(device=0, flags=flags)
        got = eng.scan_aggregate(handle, [SstInput(id=next(_ids), data=d) for d in datas], preds, **kw)
        st = eng.stats()
        eng.close()
        if fused:
            assert st["path"] == 1, "expected the fused path"
        _check(got, exp, kw["ts_col"] >= 0)
        res.append((got, st))
    (g0, s0), (g1, s1) = res
    assert g0.equals(g1)
    assert s0["rows_filtered"] == s1["rows_filtered"] and s0["rows_out"] == s1["rows_out"]
    return s0, s1


KW = dict(group_col=0, ts_col=1, window_ms=3_600_000, value_col=2)
KW_SERIES = dict(group_col=0, ts_col=-1, window_ms=0, value_col=2)


def _tags(n, pattern, rng):
    tag = rng.integers(0, 3, n).astype(np.int64)          # never 3
    if pattern == "first":
        tag[0] = 3
    elif pattern == "last":
        tag[-1] = 3
    elif pattern == "all":
        tag[:] = 3
    elif pattern == "random":
        tag[rng.random(n) < 0.3] = 3
    return tag


@pytest.mark.parametrize("rg", [1, 31, 33, 64, 8191, 8192])
@pytest.mark.parametrize("pattern", ["first", "last", "none", "all", "random"])
def test_gate_bits_row_group_shapes(rg, pattern):
    """Passing rows only at a row group's first or last row, nowhere, everywhere, at random, for row-group sizes around 32 and 8192."""
    rng = np.random.default_rng(rg * 7 + len(pattern))
    schema = _schema(pa.uint32())
    n = rg * 3 if rg >= 64 else 400
    datas = []
    for f in range(2):
        sid, ts, value = _rows(n, 17, 100 * f, rng)
        # the pattern per row group: rows are row-group aligned inside the file
        tag = np.concatenate([_tags(min(rg, n - s), pattern, rng) for s in range(0, n, rg)])
        datas.append(_write(schema, sid, ts, value, tag, rg, SNAPPY, 700 + f))
    for kw in (KW, KW_SERIES):
        _run(schema, datas, [("tag", "eq", 3)], kw, fused=rg >= 97)


@pytest.mark.parametrize("gate_type,lo,hi", [(pa.int32(), -5, 40), (pa.uint32(), 7, 4_000_000_000), (pa.int64(), -(1 << 40), 1 << 35),
                                             (pa.uint64(), 1 << 20, (1 << 63) + 5), (pa.float32(), -0.5, 0.25), (pa.float64(), -1.5, 2.0)])
@pytest.mark.parametrize("nullable", [True, False])
def test_gate_bits_types_and_levels(gate_type, lo, hi, nullable):
    """4- and 8-byte gates, signed, unsigned and floating, behind a level prefix (optional column) or none (required).  Float predicates
    run in the general pipeline: they are checked against the oracle all the same."""
    rng = np.random.default_rng(5)
    schema = _schema(gate_type, nullable)
    n = 3 * 8192 + 77
    sid, ts, value = _rows(n, 40, 0, rng)
    if pa.types.is_floating(gate_type):
        tag = rng.random(n) * 6 - 3
    elif pa.types.is_signed_integer(gate_type):
        w = 31 if gate_type == pa.int32() else 41
        tag = rng.integers(-(1 << w), 1 << w, n)
        tag[rng.random(n) < 0.2] = lo + 1
    else:
        tag = rng.integers(0, 1 << (32 if gate_type == pa.uint32() else 63), n, dtype=np.uint64)
        tag[rng.random(n) < 0.2] = lo + 3
        tag[rng.random(n) < 0.1] = np.uint64(hi - 1)
    datas = [_write(schema, sid, ts, value, tag, 8192, SNAPPY, 800)]
    fused = not pa.types.is_floating(gate_type)
    _run(schema, datas, [("tag", "ge", lo), ("tag", "lt", hi)], KW, fused=fused)


def test_gate_bits_gate_is_ts_or_value():
    """A gate column with another use: the time column (pk1, also the bucket; its sweeps read the bits, everything else its values), and
    the value column."""
    rng = np.random.default_rng(9)
    schema = _schema(pa.uint32())
    n = 5 * 8192
    sid, ts, value = _rows(n, 30, 0, rng)
    datas = [_write(schema, sid, ts, value, rng.integers(0, 5, n), 8192, SNAPPY, 810)]
    t0 = sstgen.T0_MS
    _run(schema, datas, [("ts", "ge", t0 + 3_000_000), ("ts", "lt", t0 + 30_000_000)], KW)
    _run(schema, datas, [("ts", "ge", t0 + 3_000_000), ("ts", "lt", t0 + 30_000_000)], KW_SERIES)
    # a predicate on the value column: the general pipeline (float), checked all the same
    _run(schema, datas, [("tag", "eq", 2), ("value", "ge", 10.0)], KW, fused=False)


def test_gate_bits_mixed_chunks_in_one_call():
    """Snappy, uncompressed and stored (literal-only) gate chunks in one call: the gate bits come from wherever the values are."""
    rng = np.random.default_rng(11)
    schema = _schema(pa.uint32())
    datas = []
    for f, comp in enumerate((SNAPPY, NONE, SNAPPY, NONE)):
        n = 2 * 8192 + 1000 * f
        sid, ts, value = _rows(n, 25, 100 * f, rng)
        if f == 2:
            tag = rng.integers(0, 1 << 32, n, dtype=np.uint64)    # incompressible: stored pages
            tag[rng.random(n) < 0.3] = 3
        else:
            tag = _tags(n, "random", rng)
        datas.append(_write(schema, sid, ts, value, tag, 8192, comp, 820 + f))
    for kw in (KW, KW_SERIES):
        _run(schema, datas, [("tag", "eq", 3)], kw)


def test_gate_bits_items_not_on_32_row_boundaries():
    """Work items start at key-run boundaries: series whose lengths are not multiples of 32, and a pass pattern that changes inside
    every 32-row word."""
    rng = np.random.default_rng(13)
    schema = _schema(pa.uint32())
    lens = rng.integers(1, 300, 400)
    sid = np.repeat(np.arange(len(lens)), lens)
    n = len(sid)
    ts = sstgen.T0_MS + np.arange(n) * 1000
    tag = np.where((np.arange(n) % 7) < 3, 3, 1)
    datas = [_write(schema, sid, ts, rng.random(n), tag, 8192, SNAPPY, 830)]
    for kw in (KW, KW_SERIES):
        _run(schema, datas, [("tag", "eq", 3)], kw)


def test_gate_bits_launches():
    """On resident SSTs a gated Snappy call adds three launches to the ungated call (the gate column's decompression, the row-group gate,
    the row-group compaction): the row-group gate finds the gate column's values itself, with no separate base-pointer pass."""
    rng = np.random.default_rng(17)
    schema = _schema(pa.uint32())
    n = 4 * 8192
    sid, ts, value = _rows(n, 30, 0, rng)
    data = _write(schema, sid, ts, value, _tags(n, "random", rng), 8192, SNAPPY, 840)
    handle = SchemaHandle(schema.arrow_schema, 2)
    exp = oracle.scan_aggregate([data], schema.arrow_schema, 2, [("tag", "eq", 3)], **KW)
    launches = []
    for flags in (0, HG_FLAG_NO_LATE_MATERIALIZATION):
        eng = Engine(device=0, flags=flags)
        sst_id = next(_ids)
        eng.load_sst(handle, SstInput(id=sst_id, data=data))
        got = eng.scan_aggregate(handle, [SstInput(id=sst_id, num_rows=n)], [("tag", "eq", 3)], **KW)
        st = eng.stats()
        eng.close()
        assert st["path"] == 1
        _check(got, exp, True)
        launches.append(st["kernel_launches"])
    assert launches[0] == launches[1] + 3, launches
