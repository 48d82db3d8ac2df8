"""Value mode of the Snappy decoder on the GPU (snappy_pages_kernel on INT64 / DOUBLE pages): 8-byte columns of the shapes value mode
takes, splits and refuses, written into Snappy SSTs and read back through the general pipeline (against pyarrow), and the fused
scan-aggregate on resident and transient SSTs (against the CPU oracle).  tests/test_snappy_value_mode_emu.py checks the same shapes
lane by lane on the CPU."""
import io
import itertools

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import HG_FLAG_NO_FUSED, Engine, SchemaHandle, SstInput
from horaedb_b200.config import ParquetCompression, WriteConfig
from horaedb_b200.types import StorageSchema
from oracle import oracle

pytestmark = pytest.mark.gpu
_ids = itertools.count(7100)


def _columns(n):
    rng = np.random.default_rng(31)
    t0 = 1_700_000_000_000
    base = np.arange(n, dtype=np.int64)
    cols = {
        "jitter_ts": t0 + base * 1000 + rng.integers(0, 500, n),                        # literal 1-2 + copy at offset 8 / 8 000
        "series_ts": t0 + np.tile(np.arange(1000), n // 1000 + 1)[:n] * 1000 + rng.integers(0, 200, n),
        "far_ts": t0 + np.tile(np.arange(8000), n // 8000 + 1)[:n] * 1000 + rng.integers(0, 200, n),   # sources 64 000 bytes back
        "lit3": t0 + base * 1000 + rng.integers(0, 1 << 20, n),                          # three literal bytes per value
        "lit4": t0 + base * 1000 + rng.integers(0, 1 << 28, n),
        "lit7": rng.integers(0, 1 << 55, n),                                              # no pairs: word / run mode
        "chain": t0 + base // 64,                                                         # long runs of equal values
        "spans": np.where(rng.random(n) < 0.02, 5, t0 + base * 1000 + rng.integers(0, 100, n)),
        "f64": np.cumsum(rng.integers(0, 1000, n)).astype(np.float64),
    }
    cols["mixed"] = cols["jitter_ts"].copy()
    cols["mixed"][n // 3: n // 3 + 500] = rng.integers(0, 1 << 62, 500)                 # incompressible stretch: a long literal
    return {k: (v.astype(np.float64) if k == "f64" else v.astype(np.int64)) for k, v in cols.items()}


@pytest.mark.parametrize("nullable", [False, True])
def test_general_pipeline_matches_pyarrow(nullable):
    """Row groups of 8 192, 50 000 and 777 rows: the level prefix of a nullable column's page is 8, 8 and 7 bytes (values start at
    phase 0 or 7), a required column has none; the nullable variant also carries nulls."""
    n = 50_000
    cols = _columns(n)
    names = list(cols)
    rng = np.random.default_rng(32)
    arrays = []
    for c in names:
        mask = (rng.random(n) < 0.03) if nullable else None
        arrays.append(pa.array(cols[c], mask=mask))
    spec = pa.schema([pa.field("k0", pa.uint64(), nullable=False), pa.field("k1", pa.int64(), nullable=False)] +
                     [pa.field(c, pa.float64() if c == "f64" else pa.int64(), nullable=nullable) for c in names])
    schema = StorageSchema.try_new(spec, 2)
    batch = pa.RecordBatch.from_arrays([pa.array(np.arange(n, dtype=np.uint64)), pa.array(np.zeros(n, dtype=np.int64))] + arrays, schema=spec)
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    for rg in (8192, 50_000, 777):
        data = sstgen.write_sst(schema, batch, seq=700, cfg=WriteConfig(compression=ParquetCompression.Snappy, max_row_group_size=rg), presorted=True)
        got = eng.scan(handle, [SstInput(id=next(_ids), data=data)]).read_all()
        ref = pq.read_table(io.BytesIO(data))
        for c in ["k0"] + names:
            assert got[c].to_pylist() == ref[c].to_pylist(), (rg, c)
    eng.close()


def _check(got, exp):
    assert got.num_rows == len(exp.count) > 0
    assert got["series_id"].to_numpy().tolist() == exp.gkey.tolist()
    assert got["count"].to_numpy().tolist() == exp.count.tolist()
    assert np.array_equal(got["sum"].to_numpy(), exp.sum)
    assert np.array_equal(got["min"].to_numpy(), exp.min) and np.array_equal(got["max"].to_numpy(), exp.max)


@pytest.mark.parametrize("resident", [False, True])
def test_fused_scan_resident_and_transient(resident):
    """The benchmark's query shape on Snappy SSTs: the ts pages go through value mode, decoded up to the last gate-passing row
    (partial decode), and the fused kernel's aggregate equals the oracle's; the general pipeline agrees."""
    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    datas = [sstgen.synth_sst(lo, lo + 300, 1000, 1000, seq=800 + i)[0] for i, lo in enumerate((0, 300))]
    t0 = sstgen.T0_MS
    kw = dict(group_col=0, ts_col=-1, window_ms=0, value_col=2)
    for preds in ([("tag", "eq", 3), ("ts", "ge", t0 + 250_000), ("ts", "lt", t0 + 750_000)], [("ts", "ge", t0 + 10_000)]):
        exp = oracle.scan_aggregate(datas, schema.arrow_schema, 2, preds, **kw)
        for flags in (0, HG_FLAG_NO_FUSED):
            eng = Engine(device=0, flags=flags)
            ids = [next(_ids) for _ in datas]
            if resident:
                for i, d in zip(ids, datas):
                    eng.load_sst(handle, SstInput(id=i, data=d))
                inputs = [SstInput(id=i) for i in ids]
            else:
                inputs = [SstInput(id=i, data=d) for i, d in zip(ids, datas)]
            got = eng.scan_aggregate(handle, inputs, preds, **kw)
            st = eng.stats()
            assert st["path"] == (0 if flags else 1)
            assert flags or st["decomp_ms"] > 0                   # the fused path times its decompression stage
            _check(got, exp)
            eng.close()
