"""The row-group gate of a gate-first fused scan over a 4-byte gate column, taken straight from the gate column's Snappy pages
(snappy.cu: snappy_gate_kernel; the decoder's bit domain in snappy_core.h): the column is not decompressed, its bits stand for it
everywhere.  Checked against the oracle and, bit for bit, against the same call under HG_FLAG_NO_LATE_MATERIALIZATION (no gate-first
job, the gate column decompressed and tested value by value)."""
import numpy as np
import pyarrow as pa
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import HG_FLAG_NO_LATE_MATERIALIZATION, Engine, SchemaHandle, SstInput
from oracle import oracle

from test_gpu_gate_bits import KW, KW_SERIES, SNAPPY, _check, _rows, _schema, _tags, _write

pytestmark = pytest.mark.gpu
_ids = iter(range(90_000_000, 100_000_000))


def _resident(schema, datas, preds, kw, flags):
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0, flags=flags)
    inputs = []
    for d, n in datas:
        sst_id = next(_ids)
        eng.load_sst(handle, SstInput(id=sst_id, data=d))
        inputs.append(SstInput(id=sst_id, num_rows=n))
    got = eng.scan_aggregate(handle, inputs, preds, **kw)
    st = eng.stats()
    eng.close()
    return got, st


@pytest.mark.parametrize("gate_type,tags,extra", [(pa.uint32(), "runs", 2), (pa.uint32(), "random", 3), (pa.uint64(), "runs", 3)])
def test_gate_launches_by_width_and_density(gate_type, tags, extra):
    """On resident SSTs a gated Snappy call adds launches to the ungated call: two for a run-coded 4-byte gate column (the row-group gate
    straight from its compressed pages, the row-group compaction), three for any other (the gate column's decompression, the row-group
    gate, the compaction).  A 4-byte column with a new value every few rows has too many Snappy elements per page for the bit domain."""
    rng = np.random.default_rng(17)
    schema = _schema(gate_type)
    n = 4 * 8192
    sid, ts, value = _rows(n, 30, 0, rng)
    tag = sid % 5 if tags == "runs" else _tags(n, "random", rng)
    data = _write(schema, sid, ts, value, tag, 8192, SNAPPY, 840)
    exp = oracle.scan_aggregate([data], schema.arrow_schema, 2, [("tag", "eq", 3)], **KW)
    launches = []
    for flags in (0, HG_FLAG_NO_LATE_MATERIALIZATION):
        got, st = _resident(schema, [(data, n)], [("tag", "eq", 3)], KW, flags)
        assert st["path"] == 1
        _check(got, exp, True)
        launches.append(st["kernel_launches"])
    assert launches[0] == launches[1] + extra, launches


@pytest.mark.parametrize("preds", ["config2", "tag_range", "no_match", "all_match"])
def test_config2_shape_bit_for_bit(preds):
    """Config 2's shape (the benchmark: tag = series_id mod 16 in runs of 1 000 rows, nullable; PK-disjoint files; `tag = 3 AND ts in
    [t0 + 250 s, t0 + 750 s)`, sum / count per series) resident, on a smaller scale, with the tag predicate varied."""
    t0 = sstgen.T0_MS
    ts_preds = [("ts", "ge", t0 + 250_000), ("ts", "lt", t0 + 750_000)]
    P = {"config2": [("tag", "eq", 3)] + ts_preds, "tag_range": [("tag", "ge", 5), ("tag", "lt", 9)] + ts_preds,
         "no_match": [("tag", "eq", 16)] + ts_preds, "all_match": [("tag", "lt", 16)] + ts_preds}[preds]
    schema = sstgen.metric_storage_schema()
    datas = [sstgen.synth_sst(lo, lo + 160, 1000, 1000, seq=900 + i) for i, lo in enumerate((0, 160, 320))]
    exp = oracle.scan_aggregate([d for d, _ in datas], schema.arrow_schema, 2, P, **KW_SERIES)
    (g0, s0), (g1, s1) = (_resident(schema, datas, P, KW_SERIES, f) for f in (0, HG_FLAG_NO_LATE_MATERIALIZATION))
    assert s0["path"] == 1 and s1["path"] == 1
    _check(g0, exp, False)
    assert g0.equals(g1)
    for c in ("count", "sum", "min", "max"):
        assert g0[c].to_numpy().tobytes() == g1[c].to_numpy().tobytes()
    assert s0["rows_filtered"] == s1["rows_filtered"] and s0["rows_out"] == s1["rows_out"]
