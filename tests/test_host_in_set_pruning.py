"""CPU test: row-group pruning by a sorted set (hg_plan_row_groups with HG_OP_IN_SET, host only) on pyarrow-written SSTs.

The rewrite of `col IN_SET (..)` over a chunk's statistics, computed here from pyarrow's reading of them: false when every value of the
chunk is NULL, true without statistics, else "some member of the set lies in [min, max]".  Pruning never drops a row group that holds a
member, equals HG_OP_IN's pruning for lists HG_OP_IN accepts, and the binding's argument checks."""
import ctypes as C
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from horaedb_b200 import _ffi
from horaedb_b200._ffi import HgError, HgPredicate, SchemaHandle, plan_row_groups

TYPES = [pa.uint8(), pa.int8(), pa.uint16(), pa.int16(), pa.uint32(), pa.int32(), pa.uint64(), pa.int64()]


def _bounds(t):
    bits = t.bit_width
    return (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if pa.types.is_signed_integer(t) else (0, (1 << bits) - 1)


def _file(rng, t, n, rg, null_rate, sort, span):
    lo, hi = _bounds(t)
    base = int(rng.integers(0, 3)) * ((hi - lo) // 3) + lo if hi - lo > span else lo
    vals = [min(hi, base + int(v)) for v in rng.integers(0, min(span, hi - lo) + 1, n)]
    if sort:
        vals.sort()
    v = [None if rng.random() < null_rate else x for x in vals]
    if null_rate and n > rg:
        v[:rg] = [None] * rg                                     # an all-NULL chunk
    schema = pa.schema([("pk1", pa.uint64()), ("c", t), ("f", pa.float64()), ("__seq__", pa.uint64()), ("__reserved__", pa.uint64())])
    tbl = pa.table({"pk1": pa.array(range(n), pa.uint64()), "c": pa.array(v, t), "f": pa.array(rng.random(n)), "__seq__": pa.array([1] * n, pa.uint64()),
                    "__reserved__": pa.array([None] * n, pa.uint64())}, schema=schema)
    sink = io.BytesIO()
    pq.write_table(tbl, sink, row_group_size=rg, use_dictionary=bool(rng.integers(0, 2)), compression="snappy")
    return sink.getvalue(), v, SchemaHandle(schema, 1)


def _rewrite(md, g, values):
    rgm = md.row_group(g)
    s = rgm.column(1).statistics
    if s is not None and s.has_null_count and s.null_count == rgm.num_rows:
        return 0
    if s is None or not s.has_min_max:
        return 1
    return int(any(s.min <= x <= s.max for x in values))


@pytest.mark.parametrize("t", TYPES, ids=str)
def test_in_set_pruning_is_the_rewrite_over_pyarrow_statistics(t):
    rng = np.random.default_rng(t.bit_width + 100 * pa.types.is_signed_integer(t))
    lo, hi = _bounds(t)
    for case in range(12):
        n, rg = int(rng.integers(50, 3000)), int(rng.integers(20, 400))
        data, v, handle = _file(rng, t, n, rg, [0.0, 0.3][case % 2], sort=case % 3 != 0, span=int(rng.choice([40, 5000, 1 << 40])))
        md = pq.ParquetFile(io.BytesIO(data)).metadata
        live = [x for x in v if x is not None]
        for size in (0, 1, 5, 64, 65, 700):
            values = [live[int(i)] + int(rng.integers(-2, 3)) for i in rng.integers(0, len(live), size)] if live else list(range(size))
            values = [min(hi, max(lo, x)) for x in values] + ([lo, hi] if size == 5 else [])
            rng.shuffle(values)
            keep = plan_row_groups(handle, data, [("c", "in_set", values)])
            assert keep == [_rewrite(md, g, values) for g in range(md.num_row_groups)], (case, size)
            assert keep == plan_row_groups(handle, data, [("c", "in_set", np.array(sorted(set(values)), dtype=np.int64 if lo < 0 else np.uint64))])
            members = set(values)
            for g in range(md.num_row_groups):                   # no row group holding a member is ever dropped
                if any(x in members for x in v[g * rg:(g + 1) * rg] if x is not None):
                    assert keep[g] == 1
            if len(values) <= 64:                                # HG_OP_IN's pruning, statistics only (the file has no bloom filter)
                assert keep == plan_row_groups(handle, data, [("c", "in", values)])
            both = plan_row_groups(handle, data, [("c", "in_set", values), ("pk1", "lt", n // 2)])
            assert both == [a & b for a, b in zip(keep, plan_row_groups(handle, data, [("pk1", "lt", n // 2)]))]


def test_in_set_large_sets_plan_fast_and_exactly():
    """100 000 and 2^20 values against a file of 200 row groups: the array crosses the binding without a Python loop"""
    rng = np.random.default_rng(5)
    data, v, handle = _file(rng, pa.uint64(), 20_000, 100, 0.0, sort=True, span=1 << 40)
    md = pq.ParquetFile(io.BytesIO(data)).metadata
    for size in (100_000, 1 << 20):
        values = (np.uint64(min(v)) + rng.integers(0, 1 << 39, size).astype(np.uint64))      # the lower half of the file's range
        sv = np.sort(values)
        want = []
        for g in range(md.num_row_groups):
            s = md.row_group(g).column(1).statistics
            i = np.searchsorted(sv, np.uint64(s.min))
            want.append(int(i < len(sv) and int(sv[i]) <= s.max))
        assert plan_row_groups(handle, data, [("c", "in_set", values)]) == want
        assert 0 < sum(want) < len(want)


def test_in_set_argument_checks():
    rng = np.random.default_rng(7)
    data, v, handle = _file(rng, pa.int32(), 100, 50, 0.0, True, 40)
    for col in ("f",):
        with pytest.raises(HgError) as ei:
            plan_row_groups(handle, data, [(col, "in_set", [1])])
        assert ei.value.code == 2 and "'f'" in str(ei.value)
    with pytest.raises(HgError):
        plan_row_groups(handle, data, [("c", "in_set", [1.5])])
    with pytest.raises(HgError):
        plan_row_groups(handle, data, [("c", "in_set", np.array([1.0, 2.0]))])
    L = _ffi.lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    keep, n = (C.c_uint8 * 16)(), C.c_uint32()

    def raw(op, count, ptr):
        p = (HgPredicate * 1)()
        p[0].column, p[0].op, p[0].in_count = 1, op, count
        p[0].in_values = ptr
        return L.hg_plan_row_groups(C.byref(handle.desc), C.c_void_p(buf.ctypes.data), C.c_uint64(buf.nbytes), p, C.c_size_t(1), keep, C.c_uint32(16), C.byref(n))

    one = (C.c_uint64 * 1)(1)
    assert raw(7, 1, one) == 0
    assert raw(7, 0, None) == 0 and list(keep[:2]) == [0, 0]     # the empty set matches nothing
    assert raw(7, _ffi.HG_MAX_IN_SET + 1, one) == 1              # refused before a value is read
    assert raw(7, 1, None) == 1
    assert raw(8, 1, one) != 0
    assert raw(6, 65, one) == 1                                  # HG_OP_IN keeps its limit of 64
    assert L.hg_abi_version() == 8
