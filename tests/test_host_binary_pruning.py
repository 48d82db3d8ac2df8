"""CPU test: row-group pruning by Binary statistics (hg_plan_row_groups, host only) on pyarrow-written SSTs.

PruningPredicate's rewrite over a Binary chunk's min_value / max_value: `CASE WHEN null_count = row_count THEN false ELSE <min/max
rewrite> END`, the bounds compared in arrow-rs BinaryArray order (unsigned bytes, a proper prefix first; Python's bytes order is the
same).  min_value / max_value are bounds, so `<>` never prunes, and pruning never drops a row group that holds a passing row.  Also the
argument checks of Binary predicates."""
import ctypes as C
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from horaedb_b200 import _ffi
from horaedb_b200._ffi import HgBytes, HgError, HgPredicate, SchemaHandle, plan_row_groups

SCHEMA = pa.schema([("pk1", pa.uint64()), ("b", pa.binary()), ("c", pa.binary()), ("__seq__", pa.uint64()), ("__reserved__", pa.uint64())])
HANDLE = SchemaHandle(SCHEMA, 1)
HOLDS = {"eq": lambda v, x: v == x, "ne": lambda v, x: v != x, "lt": lambda v, x: v < x, "le": lambda v, x: v <= x, "gt": lambda v, x: v > x,
         "ge": lambda v, x: v >= x}
ALPHABET = [b"", b"\x00", b"\x01", b"a", b"ab", b"\x7f", b"\x80", b"\xff", b"prefix08", b"prefix16prefix16"]


def _value(rng):
    k = rng.random()
    if k < 0.4:                                              # short strings over a tiny alphabet: many ties and prefixes
        return b"".join(ALPHABET[int(i)] for i in rng.integers(0, len(ALPHABET), int(rng.integers(0, 4))))
    if k < 0.5:
        return b"\xff" * int(rng.integers(7, 11))
    return bytes(rng.integers(0, 256, int(rng.integers(0, 20)), dtype=np.uint8))


def _file(rng, n, rg, null_rate, sort):
    b = [None if rng.random() < null_rate else _value(rng) for _ in range(n)]
    if sort:
        b = sorted(v for v in b if v is not None) + [None] * sum(v is None for v in b)
    c = [_value(rng) for _ in range(n)]
    t = pa.table({"pk1": pa.array(range(n), pa.uint64()), "b": pa.array(b, pa.binary()), "c": pa.array(c, pa.binary()),
                  "__seq__": pa.array([1] * n, pa.uint64()), "__reserved__": pa.array([None] * n, pa.uint64())})
    sink = io.BytesIO()
    pq.write_table(t, sink, row_group_size=rg, use_dictionary=bool(rng.integers(0, 2)), compression="snappy")
    return sink.getvalue(), b, c


def _rewrite(md, g, col, op, lits):
    """the rewrite from pyarrow's reading of the chunk statistics"""
    rgm = md.row_group(g)
    s = rgm.column(col).statistics
    if s is not None and s.has_null_count and s.null_count == rgm.num_rows:
        return 0
    if s is None or not s.has_min_max or op == "ne":
        return 1
    if op == "in":
        return int(any(s.min <= x <= s.max for x in lits))
    x = lits
    return int({"eq": s.min <= x <= s.max, "lt": s.min < x, "le": s.min <= x, "gt": s.max > x, "ge": s.max >= x}[op])


def _literal(rng, vals):
    live = [v for v in vals if v is not None]
    k = rng.random()
    if k < 0.4 and live:
        return live[int(rng.integers(0, len(live)))]
    if k < 0.6 and live:
        v = live[int(rng.integers(0, len(live)))]
        return v[:int(rng.integers(0, len(v) + 1))] + (b"" if rng.random() < 0.5 else bytes([int(rng.integers(0, 256))]))
    return _value(rng)


@pytest.mark.parametrize("seed", range(6))
def test_random_tables_and_literals(seed):
    rng = np.random.default_rng(900 + seed)
    for sort in (True, False):
        data, b, c = _file(rng, 1200, int(rng.integers(40, 300)), (0.0, 0.2, 0.97)[seed % 3], sort)
        md = pq.ParquetFile(io.BytesIO(data)).metadata
        bounds = [0]
        for g in range(md.num_row_groups):
            bounds.append(bounds[-1] + md.row_group(g).num_rows)
        pruned = 0
        for _ in range(60):
            op = ["eq", "ne", "lt", "le", "gt", "ge", "in"][int(rng.integers(0, 7))]
            lits = [_literal(rng, b) for _ in range(int(rng.integers(0, 9)))] if op == "in" else _literal(rng, b)
            keep = plan_row_groups(HANDLE, data, [("b", op, lits)])
            assert keep == [_rewrite(md, g, 1, op, lits) for g in range(md.num_row_groups)], (op, lits)
            for g in range(md.num_row_groups):
                rows = b[bounds[g]:bounds[g + 1]]
                passing = any(v is not None and (any(v == x for x in lits) if op == "in" else HOLDS[op](v, lits)) for v in rows)
                assert keep[g] or not passing, (g, op, lits)
                pruned += 1 - keep[g]
            if op == "ne":
                assert keep == [int(md.row_group(g).column(1).statistics.null_count < md.row_group(g).num_rows) for g in range(md.num_row_groups)]
        if sort and seed % 3 != 2:
            assert pruned > 0
        # a conjunction over both Binary columns = the AND of the two rewrites
        x, y = _literal(rng, b), _literal(rng, c)
        want = [_rewrite(md, g, 1, "ge", x) & _rewrite(md, g, 2, "lt", y) for g in range(md.num_row_groups)]
        assert plan_row_groups(HANDLE, data, [("b", "ge", x), ("c", "lt", y)]) == want


def test_not_equal_never_prunes_and_prefix_order():
    vals = [b"", b"\x00", b"ab", b"ab\x00", b"abc", b"\xff"]           # one value per row group, in BinaryArray order
    t = pa.table({"pk1": pa.array(range(6), pa.uint64()), "b": pa.array(vals, pa.binary()), "c": pa.array(vals, pa.binary()),
                  "__seq__": pa.array([1] * 6, pa.uint64()), "__reserved__": pa.array([None] * 6, pa.uint64())})
    sink = io.BytesIO()
    pq.write_table(t, sink, row_group_size=1)
    data = sink.getvalue()
    for i, x in enumerate(vals):
        assert plan_row_groups(HANDLE, data, [("b", "ne", x)]) == [1] * 6
        assert plan_row_groups(HANDLE, data, [("b", "eq", x)]) == [int(j == i) for j in range(6)]
        assert plan_row_groups(HANDLE, data, [("b", "lt", x)]) == [int(j < i) for j in range(6)]
        assert plan_row_groups(HANDLE, data, [("b", "ge", x)]) == [int(j >= i) for j in range(6)]
    assert plan_row_groups(HANDLE, data, [("b", "in", [])]) == [0] * 6
    assert plan_row_groups(HANDLE, data, [("b", "in", [b"ab\x00", b"ab\x00", b"zz"])]) == [0, 0, 0, 1, 0, 0]
    assert plan_row_groups(HANDLE, data, [("b", "eq", b"ab"), ("b", "eq", b"abc")]) == [0] * 6
    assert plan_row_groups(HANDLE, data, [("b", "eq", bytearray(b"ab")), ("c", "gt", memoryview(b"a"))]) == [0, 0, 1, 0, 0, 0]


def _raw_plan(preds):
    arr = (HgPredicate * len(preds))(*preds)
    keep = (C.c_uint8 * 64)()
    n = C.c_uint32()
    data = np.frombuffer(_file(np.random.default_rng(1), 50, 10, 0.0, True)[0], dtype=np.uint8)
    return _ffi.lib().hg_plan_row_groups(C.byref(HANDLE.desc), C.c_void_p(data.ctypes.data), C.c_uint64(data.nbytes), arr, C.c_size_t(len(preds)),
                                         keep, C.c_uint32(64), C.byref(n))


def test_invalid_binary_predicates():
    one = (HgBytes * 1)(HgBytes(None, 0))
    ok = HgPredicate(column=1, op=0)
    ok.in_bytes, ok.in_count = one, 1
    assert _raw_plan([ok]) == 0                                          # b = b"": a null pointer with length 0 is a valid literal
    null_list = HgPredicate(column=1, op=0)
    null_list.in_count = 1
    assert _raw_plan([null_list]) == 1                                   # null in_bytes
    null_in = HgPredicate(column=1, op=6)
    assert _raw_plan([null_in]) == 1                                     # ... for IN too, even with no literal
    bad_data = (HgBytes * 1)(HgBytes(None, 3))
    p = HgPredicate(column=1, op=2)
    p.in_bytes, p.in_count = bad_data, 1
    assert _raw_plan([p]) == 1                                           # null data, len > 0
    for op in range(6):
        p = HgPredicate(column=1, op=op)
        p.in_bytes, p.in_count = one, 0
        assert _raw_plan([p]) == 1                                       # a comparison without its literal
        p.in_count = 2
        assert _raw_plan([p]) == 1                                       # ... or with two
    for preds in ([("b", "in", [b"x"] * 65)], [("b", "eq", b"x" * 65_537)], [("b", "in", [b"", b"y" * 65_537])]):
        with pytest.raises(HgError) as ei:
            plan_row_groups(HANDLE, _file(np.random.default_rng(2), 20, 10, 0.0, True)[0], preds)
        assert ei.value.code == 1
    assert len(plan_row_groups(HANDLE, _file(np.random.default_rng(2), 20, 10, 0.0, True)[0], [("b", "in", [b"x"] * 64), ("b", "le", b"y" * 65_536)])) == 2
    for lit in (1, 1.5, "abc", None, [b"a"]):
        with pytest.raises(HgError) as ei:
            plan_row_groups(HANDLE, _file(np.random.default_rng(3), 20, 10, 0.0, True)[0], [("b", "eq", lit)])
        assert ei.value.code == 1
    with pytest.raises(HgError) as ei:
        plan_row_groups(HANDLE, _file(np.random.default_rng(3), 20, 10, 0.0, True)[0], [("b", "in", b"ab")])
    assert ei.value.code == 1
