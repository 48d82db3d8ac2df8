"""The fused aggregate's shape (fused_scan.cu: fused_shape) decides both whether the fused kernel runs and whether a transient load may ship
compressed prefixes of the pages that kernel reads only up to the gate's last passing row.  A call the fused kernel refuses for its shape
(pk0 a 4-byte integer) runs on the general pipeline, which decodes whole pages: its transient load must ship whole pages, so the call runs
once, never repeated for a prefix that ran out."""
import numpy as np
import pyarrow as pa
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import HG_FLAG_NO_LATE_MATERIALIZATION, Engine, SchemaHandle, SstInput
from horaedb_b200.config import ParquetCompression, WriteConfig
from horaedb_b200.types import StorageSchema
from oracle import oracle

pytestmark = pytest.mark.gpu
_ids = iter(range(90_000_000, 91_000_000))


def test_transient_call_with_an_unfusable_shape_ships_whole_pages():
    fields = [pa.field("series_id", pa.int32(), False), pa.field("ts", pa.int64(), False), pa.field("value", pa.float64(), False),
              pa.field("tag", pa.uint32(), False)]
    schema = StorageSchema.try_new(pa.schema(fields), 2)
    rng = np.random.default_rng(33)
    n = 40_000
    sid = np.repeat(np.arange(-20, 20), 1000).astype(np.int32)
    ts = sstgen.T0_MS + np.tile(np.arange(1000) * 1000 + rng.integers(0, 400, 1000), 40)
    # 8192-row groups: in the first three the passing rows sit in the first half; the last two pass none, though their statistics
    # (2 .. 4) cannot tell, so the gate column prunes them
    i = np.arange(n)
    tag = np.where(i < 3 * 8192, np.where(i % 8192 < 3500, 3, 5), 2 + 2 * (i % 2)).astype(np.uint32)
    value = np.round(rng.random(n), 2)                                       # compressible: its Snappy pages are no stored pages
    batch = pa.RecordBatch.from_arrays([pa.array(sid), pa.array(ts.astype(np.int64)), pa.array(value), pa.array(tag)], schema=pa.schema(fields))
    data = sstgen.write_sst(schema, batch, seq=7, cfg=WriteConfig(compression=ParquetCompression.Snappy), presorted=True)
    handle = SchemaHandle(schema.arrow_schema, 2)
    preds = [("tag", "eq", 3)]
    kw = dict(group_col=0, ts_col=-1, window_ms=0, value_col=2)
    exp = oracle.scan_aggregate([data], schema.arrow_schema, 2, preds, **kw)
    stats = []
    for flags in (0, HG_FLAG_NO_LATE_MATERIALIZATION):
        eng = Engine(device=0, flags=flags)
        got = eng.scan_aggregate(handle, [SstInput(id=next(_ids), data=data)], preds, **kw)
        stats.append(eng.stats())
        eng.close()
        assert got["series_id"].to_numpy().tolist() == exp.gkey.astype(np.int64).tolist()     # (the oracle widens keys to 64 bits)
        assert got["count"].to_numpy().tolist() == exp.count.tolist()
        assert np.array_equal(got["sum"].to_numpy(), exp.sum)
        assert np.array_equal(got["min"].to_numpy(), exp.min) and np.array_equal(got["max"].to_numpy(), exp.max)
    assert stats[0]["path"] & 2 == 0, "the call was repeated with whole pages"
    assert stats[0]["bytes_h2d"] <= stats[1]["bytes_h2d"]
