"""Predicates, time buckets and min / max / sum at the edges of the value domain, on every path that evaluates them: the fused
aggregate on resident SSTs (gated and with HG_FLAG_NO_LATE_MATERIALIZATION) and on transient SSTs, the general pipeline in RUNS and
HASH mode, `scan`, and statistics pruning switched off.

Every answer is checked against a plain Python model written here, independent of the C oracle, and against the oracle:
  * integers are Python ints; floats compare in IEEE totalOrder on their bits (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN);
  * predicates form a conjunction, a NULL fails, IN is an OR of `=`;
  * primary keys are unique, so the stream is primary-key order and nothing is deduplicated;
  * groups are pk0 [, bucket = ts / w * w with TRUNCATING division]; count = rows, sum = sequential float sum from 0.0,
    min / max = the first non-null value, then strict `<` / `>`.
f64 results are compared by their bits, so -0.0 differs from +0.0 and a NaN's sign and payload count."""
import struct

import numpy as np
import pyarrow as pa
import pytest

from helpers import arrays_equal
from horaedb_b200._ffi import (HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_NO_FUSED, HG_FLAG_NO_LATE_MATERIALIZATION, HG_FLAG_NO_PRUNING, Engine,
                               SchemaHandle, SstInput)
from horaedb_b200 import sstgen
from horaedb_b200.config import ParquetCompression, WriteConfig
from horaedb_b200.types import StorageSchema
from oracle import oracle

pytestmark = pytest.mark.gpu
_ids = iter(range(70_000_000, 80_000_000))

I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1
INT_TYPES = {"u8": pa.uint8(), "i8": pa.int8(), "u16": pa.uint16(), "i16": pa.int16(), "u32": pa.uint32(), "i32": pa.int32(),
             "u64": pa.uint64(), "i64": pa.int64()}


def _edges(t: pa.DataType):
    """min, min+1, -1 (signed), 0, 1, max-1, max of an integer type"""
    bits = t.bit_width
    if pa.types.is_signed_integer(t):
        lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
        return [lo, lo + 1, -1, 0, 1, hi - 1, hi]
    hi = (1 << bits) - 1
    return [0, 1, 2, hi - 1, hi]


# ------------------------------------------------------------------------------------------------------------- the model
def f64_of(bits: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def bits_of(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f32_widened(bits: int) -> int:
    """f32 bits -> f64 bits, exactly; a (quiet) NaN keeps its sign and payload"""
    if (bits >> 23) & 0xFF == 0xFF and bits & 0x7FFFFF:
        return ((bits >> 31) << 63) | (0x7FF << 52) | ((bits & 0x7FFFFF) << 29)
    return bits_of(struct.unpack("<f", struct.pack("<I", bits))[0])


def sum_bits(bits: int):
    """A sum is compared by its bits unless it is a NaN.  Which NaN a sum ends with is not defined anywhere: IEEE 754 leaves the
    payload of NaN + NaN (and the sign of inf + -inf's NaN) to the implementation, and a compiler may swap the operands of an
    add; the oracle itself changes with it.  Min and max select one of the values, so their bits are always compared."""
    return "NaN" if (bits >> 52) & 0x7FF == 0x7FF and bits & ((1 << 52) - 1) else bits


def total_order_key(f64_bits: int) -> int:
    return f64_bits ^ (U64_MAX if f64_bits >> 63 else 1 << 63)


class Table:
    """Columns as Python values in stream (primary-key) order: ints, or the BITS of f32 / f64 values; None = NULL."""

    def __init__(self, user: pa.Schema, cols: dict):
        self.user, self.cols = user, cols
        self.n = len(next(iter(cols.values())))
        self.schema = StorageSchema.try_new(user, 2)
        self.handle = SchemaHandle(self.schema.arrow_schema, 2)

    def typ(self, name):
        return self.user.field(name).type

    def key(self, name, v):
        """order key of a stored value / literal in the column's comparison class (Python int)"""
        t = self.typ(name)
        if t == pa.float32():
            return total_order_key(f32_widened(v))
        if t == pa.float64():
            return total_order_key(v)
        return v

    def lit_key(self, name, lit):
        return total_order_key(bits_of(float(lit))) if pa.types.is_floating(self.typ(name)) else int(lit)

    def passes(self, r, preds):
        for name, op, lit in preds:
            v = self.cols[name][r]
            if v is None:
                return False
            k = self.key(name, v)
            if op == "in":
                if not any(k == self.lit_key(name, x) for x in lit):
                    return False
                continue
            c = self.lit_key(name, lit)
            if not {"eq": k == c, "ne": k != c, "lt": k < c, "le": k <= c, "gt": k > c, "ge": k >= c}[op]:
                return False
        return True

    def survivors(self, preds):
        return [r for r in range(self.n) if self.passes(r, preds)]

    def aggregate(self, preds, group, ts, w, value):
        """[(gkey, bucket, count, sum bits, min bits, max bits)] in (pk0, bucket) order"""
        out = []
        for r in self.survivors(preds):
            k = self.cols[group][r] if group else 0
            b = 0
            if ts and w > 0:
                t = self.cols[ts][r]
                q = abs(t) // w
                b = (q if t >= 0 else -q) * w          # truncating division, in Python ints
            if not out or out[-1][0] != k or out[-1][1] != b:
                out.append([k, b, 0, 0.0, float("inf"), float("-inf"), False])
            g = out[-1]
            g[2] += 1
            if value:
                v = self.cols[value][r]
                if v is not None:
                    x = f64_of(v)
                    g[3] += x
                    if not g[6] or x < g[4]:
                        g[4] = x
                    if not g[6] or x > g[5]:
                        g[5] = x
                    g[6] = True
        return [(k, b, c, sum_bits(bits_of(s)), bits_of(mn), bits_of(mx)) for k, b, c, s, mn, mx, _ in out]

    def batch(self):
        arrays = []
        for f in self.user:
            v = self.cols[f.name]
            mask = np.array([x is None for x in v])
            if pa.types.is_floating(f.type):
                it, ft = (np.uint32, np.float32) if f.type == pa.float32() else (np.uint64, np.float64)
                raw = np.array([0 if x is None else x for x in v], dtype=it).view(ft)
                arrays.append(pa.array(raw, f.type, mask=mask))
            else:
                arrays.append(pa.array(v, f.type))
        return pa.RecordBatch.from_arrays(arrays, schema=self.user)

    def write(self, rows_per_rg, compression=ParquetCompression.Uncompressed):
        return sstgen.write_sst(self.schema, self.batch(), seq=next(_ids) % 100_000 + 1,
                                cfg=WriteConfig(compression=compression, max_row_group_size=rows_per_rg), presorted=True)


# ------------------------------------------------------------------------------------------------------- the checks
class Runner:
    """One table's SSTs, resident in one engine, plus the host bytes for transient loads and the oracle."""

    def __init__(self, table: Table, datas):
        self.t, self.datas = table, datas
        self.eng = Engine(device=0)
        self.ids = []
        for d in datas:
            sid = next(_ids)
            self.eng.load_sst(table.handle, SstInput(id=sid, data=d))
            self.ids.append(sid)

    def close(self):
        self.eng.close()

    def _agg(self, flags, resident, preds, kw):
        self.eng.set_flags(flags)
        ins = [SstInput(id=i) for i in self.ids] if resident else [SstInput(id=next(_ids), data=d) for d in self.datas]
        got = self.eng.scan_aggregate(self.t.handle, ins, preds, **kw)
        return got, self.eng.stats()["path"]

    def rows(self, got, kw):
        """result table -> [(gkey, bucket, count, sum bits, min bits, max bits)]"""
        n = got.num_rows
        gk = got.column(0).to_pylist() if kw["group_col"] >= 0 else [0] * n
        bk = got["bucket"].to_pylist() if kw["ts_col"] >= 0 and kw["window_ms"] > 0 else [0] * n
        cnt = got["count"].to_pylist()
        if kw["value_col"] < 0:
            return [(a, b, c, 0, 0, 0) for a, b, c in zip(gk, bk, cnt)]
        s, mn, mx = [got[c].combine_chunks().to_numpy(zero_copy_only=False).view(np.uint64).tolist() if n else [] for c in ("sum", "min", "max")]
        return list(zip(gk, bk, cnt, [sum_bits(x) for x in s], mn, mx))

    def oracle_rows(self, preds, kw, prune=True):
        o = oracle.scan_aggregate(self.datas, self.t.schema.arrow_schema, 2, preds, prune=prune, **kw)
        signed = kw["group_col"] >= 0 and pa.types.is_signed_integer(self.t.user.field(kw["group_col"]).type)
        gk = [(int(x) - (1 << 64) if signed and int(x) >> 63 else int(x)) for x in o.gkey] if kw["group_col"] >= 0 else [0] * len(o.count)
        bk = o.bucket.tolist() if kw["ts_col"] >= 0 and kw["window_ms"] > 0 else [0] * len(o.count)
        if kw["value_col"] < 0:
            return [(a, b, int(c), 0, 0, 0) for a, b, c in zip(gk, bk, o.count)]
        s, mn, mx = [a.view(np.uint64).tolist() for a in (o.sum, o.min, o.max)]
        return list(zip(gk, bk, [int(c) for c in o.count], [sum_bits(x) for x in s], mn, mx))

    def model(self, preds, kw):
        names = self.t.user.names
        col = lambda i: names[i] if i >= 0 else None
        exp = self.t.aggregate(preds, col(kw["group_col"]), col(kw["ts_col"]), kw["window_ms"], col(kw["value_col"]))
        if kw["value_col"] < 0:
            exp = [(a, b, c, 0, 0, 0) for a, b, c, *_ in exp]
        if kw["group_col"] < 0 and kw["ts_col"] < 0:
            exp = [(0, 0, sum(e[2] for e in exp), 0, 0, 0)] if exp else []
        return exp

    def check_aggregate(self, preds, kw, fused=True, nan_columns=False):
        """every aggregate path against the model and the oracle; `fused`: the fused planner must take the call"""
        exp = self.model(preds, kw)
        ctx = f"preds={preds} kw={kw}"
        assert self.oracle_rows(preds, kw, prune=False) == exp, "oracle (no pruning) vs model: " + ctx
        if not nan_columns:
            assert self.oracle_rows(preds, kw) == exp, "oracle vs model: " + ctx
        pruned = self.oracle_rows(preds, kw) if nan_columns else exp
        hash_kw = dict(kw, mode=HG_AGG_HASH)
        runs = [("fused, resident", 0, True, kw, 1), ("fused, resident, no late materialisation", HG_FLAG_NO_LATE_MATERIALIZATION, True, kw, 1),
                ("fused, transient", 0, False, kw, 1), ("fused, resident, hash mode", 0, True, hash_kw, 1),
                ("general, runs", HG_FLAG_NO_FUSED, True, kw, 0), ("general, hash", HG_FLAG_NO_FUSED, True, hash_kw, 0),
                ("general, transient", HG_FLAG_NO_FUSED, False, kw, 0)]
        for name, flags, resident, k2, path in runs:
            if not fused and path == 1 and flags:
                continue                                   # (the same call as the one without the flag)
            got, p = self._agg(flags, resident, preds, k2)
            if fused:
                assert p == path, f"{name}: expected path {path}, got {p}: " + ctx
            assert self.rows(got, kw) == pruned, f"{name}: " + ctx
        for name, resident, k2 in (("no pruning", True, kw), ("no pruning, transient", False, kw)):
            got, p = self._agg(HG_FLAG_NO_PRUNING, resident, preds, k2)
            assert self.rows(got, kw) == exp, f"{name}: " + ctx
        self.eng.set_flags(0)

    def check_scan(self, preds, nan_columns=False):
        """`scan` (eval_predicates_kernel) row for row against the model, and against the oracle with the same pruning"""
        full = self.t.batch()
        ctx = f"preds={preds}"
        exp = pa.Table.from_batches([full]).take(pa.array(self.t.survivors(preds), pa.int64()))
        for flags, prune in ((0, True), (HG_FLAG_NO_PRUNING, False)):
            self.eng.set_flags(flags)
            got = self.eng.scan(self.t.handle, [SstInput(id=i) for i in self.ids], preds).read_all()
            orc = oracle.scan(self.datas, self.t.schema.arrow_schema, 2, preds, prune=prune).batches
            orc = pa.Table.from_batches(orc, schema=got.schema) if orc else got.slice(0, 0)
            want = orc if (nan_columns and prune) else exp
            assert got.num_rows == want.num_rows == orc.num_rows, f"rows {got.num_rows} / {want.num_rows} / oracle {orc.num_rows}: {ctx} flags={flags}"
            for c in range(got.num_columns):
                assert arrays_equal(got.column(c), want.column(c)), f"column {got.schema.names[c]}: {ctx} flags={flags}"
                assert arrays_equal(orc.column(c), want.column(c)), f"oracle column {got.schema.names[c]}: {ctx} flags={flags}"
        self.eng.set_flags(0)


# ------------------------------------------------------------------------------ integer predicates at the type edges
ROWS_PER_KEY = 1024


def _int_table(pk0_type):
    """pk0 (i64 or u64) at its type's edges, one row group of ROWS_PER_KEY rows per pk0 value (so that no row group's pk0 span
    wraps: the fused planner bounds the groups by it); one predicate column per integer width and signedness, each cycling
    through its type's edges at its own stride."""
    pk0 = [I64_MIN, -1, 0, I64_MAX] if pk0_type == pa.int64() else [0, I64_MAX, 1 << 63, U64_MAX]
    fields = [pa.field("k", pk0_type), pa.field("t", pa.int64()), pa.field("v", pa.float64())]
    fields += [pa.field("c_" + n, t) for n, t in INT_TYPES.items()]
    user = pa.schema([pa.field(f.name, f.type, True) for f in fields])
    rng = np.random.default_rng(5)
    n = len(pk0) * ROWS_PER_KEY
    cols = {"k": [k for k in pk0 for _ in range(ROWS_PER_KEY)],
            "t": [t for _ in pk0 for t in (-5000 + 7 * np.arange(ROWS_PER_KEY)).tolist()],
            "v": [bits_of(float(x)) for x in rng.integers(-1000, 1000, n) / 8]}
    for j, (name, t) in enumerate(INT_TYPES.items()):
        e = _edges(t)
        cols["c_" + name] = [e[(r * (j + 1) + r // 5) % len(e)] for r in range(n)]
    return Table(user, cols)


def _int_pair_cases(name, t):
    e = _edges(t)
    lo, hi = e[0], e[-1]
    mid = 0 if pa.types.is_signed_integer(t) else 1
    c = "c_" + name
    return [[(c, "eq", lo), (c, "eq", hi)],                     # contradiction
            [(c, "ge", e[-2]), (c, "le", e[1])],                # >= b AND <= a, a < b
            [(c, "lt", lo)], [(c, "gt", hi)],                   # below the minimum / above the maximum
            [(c, "ge", hi), (c, "le", hi)], [(c, "ge", lo), (c, "le", lo)],   # single points at the edges
            [(c, "ge", lo)],                                    # passes every row
            [(c, "ge", -1 if mid == 0 else 0), (c, "le", 1)],   # an interval around zero
            [(c, "gt", lo), (c, "lt", hi)]]


@pytest.fixture(scope="module", params=["i64", "u64"])
def int_runner(request):
    t = _int_table(pa.int64() if request.param == "i64" else pa.uint64())
    r = Runner(t, [t.write(ROWS_PER_KEY)])
    yield r
    r.close()


AGG_KW = dict(group_col=0, ts_col=-1, window_ms=0, value_col=2)
COUNT_KW = dict(group_col=-1, ts_col=-1, window_ms=0, value_col=-1)


def test_int_predicates_every_op_and_edge_literal(int_runner):
    """Every op with every edge literal of the column's type, on every integer width: the fused kernel's interval test (8-byte
    keys, the 32-bit rebase of 1-, 2- and 4-byte columns) against the model."""
    r = int_runner
    for name, t in INT_TYPES.items():
        for lit in _edges(t):
            for op in ("eq", "lt", "le", "gt", "ge"):
                preds = [("c_" + name, op, lit)]
                exp = r.model(preds, AGG_KW)
                for flags, resident in ((0, True), (HG_FLAG_NO_LATE_MATERIALIZATION, True), (0, False), (HG_FLAG_NO_FUSED, True)):
                    got, path = r._agg(flags, resident, preds, AGG_KW)
                    assert path == (0 if flags & HG_FLAG_NO_FUSED else 1)
                    assert r.rows(got, AGG_KW) == exp, f"preds={preds} flags={flags} resident={resident}"
    r.eng.set_flags(0)


@pytest.mark.parametrize("col", list(INT_TYPES))
def test_int_predicate_pairs_on_one_column(int_runner, col):
    """Contradictions, empty and single-point intervals, `>= min`, intervals across zero: every aggregate path, the global
    count(*) included."""
    for preds in _int_pair_cases(col, INT_TYPES[col]):
        int_runner.check_aggregate(preds, AGG_KW)
        int_runner.check_aggregate(preds, COUNT_KW)


def test_pk_edges_empty_time_range_and_two_extra_columns(int_runner):
    """Predicates on pk0 at its type's edges, the empty time range `t >= x AND t < x`, and two extra predicate columns (the
    planner makes the narrower one the gate), with and without a contradiction among them."""
    r = int_runner
    pk = sorted(set(r.t.cols["k"]))
    cases = [[("t", "ge", 100), ("t", "lt", 100)], [("t", "ge", I64_MIN), ("t", "le", I64_MAX)], [("t", "gt", I64_MAX - 1)],
             [("t", "lt", I64_MIN + 1)], [("t", "ge", -1), ("t", "le", 1)]]
    for k in pk:
        cases += [[("k", "eq", k)], [("k", "ge", k)], [("k", "lt", k)], [("k", "gt", k), ("t", "ge", 0)]]
    cases += [[("k", "eq", pk[0]), ("k", "eq", pk[-1])], [("k", "gt", pk[1]), ("k", "lt", pk[2])]]
    cases += [[("c_u8", "ge", 1), ("c_i64", "le", 0)],                      # 4-byte gate after the swap
              [("c_i64", "eq", I64_MIN), ("c_u8", "eq", 255)],              # given in the other order
              [("c_i16", "eq", -(1 << 15)), ("c_u32", "eq", (1 << 32) - 1)],
              [("c_u64", "ge", U64_MAX - 1), ("c_i8", "lt", 0), ("t", "ge", -2000)],
              [("c_u16", "eq", 1), ("c_u16", "eq", 2), ("c_i32", "ge", 0)],    # a contradiction on one of two extra columns
              [("c_i32", "ge", 1 << 30), ("c_u64", "lt", 0 + 1), ("c_u64", "gt", 0)]]
    for preds in cases:
        r.check_aggregate(preds, AGG_KW)
        r.check_aggregate(preds, COUNT_KW)


def test_int_predicates_through_scan(int_runner):
    """The same predicates through `scan` (eval_predicates_kernel), row for row; IN lists holding the extremes and an empty
    IN list (the general pipeline takes IN and `!=`)."""
    r = int_runner
    for name, t in INT_TYPES.items():
        e = _edges(t)
        c = "c_" + name
        for preds in _int_pair_cases(name, t) + [[(c, "in", [e[0], e[-1]])], [(c, "in", [])], [(c, "ne", e[0])], [(c, "ne", e[-1]), (c, "in", e)],
                                                 [(c, "in", [e[1], e[-2]]), (c, "ge", e[1])]]:
            r.check_scan(preds)
            if any(op in ("in", "ne") for _, op, _ in preds):
                r.check_aggregate(preds, AGG_KW, fused=False)
    pk = sorted(set(r.t.cols["k"]))
    r.check_scan([("k", "in", [pk[0], pk[-1]])])
    r.check_aggregate([("k", "in", [pk[0], pk[-1]])], AGG_KW, fused=False)


# ----------------------------------------------------------------------------------- float predicates, general path
F32_SPECIAL = [0xFFC00000, 0x7FC00000, 0x7FC12345, 0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x80000001,
               0x007FFFFF, 0x7F7FFFFF, 0xFF7FFFFF, 0x00800000, 0x3DCCCCCD, 0xBF800000, 0x3F800000]     # ..., 0.1f, -1, 1
F64_SPECIAL = [0xFFF8000000000000, 0x7FF8000000000000, 0x7FF8000000012345, 0, 1 << 63, 0x7FF0000000000000, 0xFFF0000000000000, 1,
               (1 << 63) | 1, 0x000FFFFFFFFFFFFF, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF, 0x0010000000000000, bits_of(0.1),
               bits_of(-1.0), bits_of(1.0)]


@pytest.fixture(scope="module")
def float_runner():
    user = pa.schema([pa.field("k", pa.uint64(), True), pa.field("t", pa.int64(), True), pa.field("v", pa.float64(), True),
                      pa.field("f32", pa.float32(), True), pa.field("f64", pa.float64(), True)])
    n, per = 1024, 256
    cols = {"k": [r // per for r in range(n)], "t": [r % per for r in range(n)],
            "v": [bits_of(float(r % 13) - 6.0) for r in range(n)],
            "f32": [F32_SPECIAL[(r * 3 + r // 16) % len(F32_SPECIAL)] for r in range(n)],
            "f64": [F64_SPECIAL[(r * 5 + r // 16) % len(F64_SPECIAL)] for r in range(n)]}
    # one row group without NaNs, so that pruning has statistics that bound every value there
    for r in range(3 * per, n):
        for c, sp in (("f32", F32_SPECIAL), ("f64", F64_SPECIAL)):
            while cols[c][r] in sp[:3]:
                cols[c][r] = sp[(sp.index(cols[c][r]) + 5) % len(sp)]
    t = Table(user, cols)
    r = Runner(t, [t.write(per)])
    yield r
    r.close()


def _float_literals():
    lits = [f64_of(b) for b in F64_SPECIAL]
    return lits + [f64_of(f32_widened(b)) for b in F32_SPECIAL if b not in (0x3DCCCCCD,)] + [0.1]


def test_float_predicates_every_op_and_special_literal(float_runner):
    """f32 and f64 columns holding NaNs of both signs and a payload NaN, signed zeros, infinities, subnormals, the extremes and
    the smallest normal, compared with the same set of literals by every op (totalOrder); the f32 column is also compared with
    0.1, which it cannot represent.  The widening of f32 on the device must equal the exact one."""
    r = float_runner
    for col in ("f32", "f64"):
        for lit in _float_literals():
            for op in ("eq", "ne", "lt", "le", "gt", "ge"):
                preds = [(col, op, lit)]
                r.check_scan(preds, nan_columns=True)
                exp = r.model(preds, AGG_KW)
                for flags, resident in ((HG_FLAG_NO_PRUNING, True), (HG_FLAG_NO_PRUNING, False)):
                    got, path = r._agg(flags, resident, preds, AGG_KW)
                    assert path == 0 and r.rows(got, AGG_KW) == exp, f"preds={preds} flags={flags} resident={resident}"
                got, _ = r._agg(0, True, preds, AGG_KW)
                assert r.rows(got, AGG_KW) == r.oracle_rows(preds, AGG_KW), f"preds={preds} (pruned like the oracle)"
    r.eng.set_flags(0)


def test_float_in_lists_and_conjunctions(float_runner):
    r = float_runner
    nan, neg_nan, pay = (f64_of(b) for b in F64_SPECIAL[:3])
    cases = [[("f64", "in", [nan, neg_nan])], [("f64", "in", [pay])], [("f64", "in", [0.0])], [("f64", "in", [-0.0, float("inf")])],
             [("f64", "in", [])], [("f32", "in", [0.1])], [("f32", "in", [f64_of(f32_widened(0x3DCCCCCD)), nan])],
             [("f32", "in", [f64_of(f32_widened(0x7FC12345)), f64_of(f32_widened(0xFFC00000))])],
             [("f64", "ge", -0.0), ("f64", "le", 0.0)], [("f64", "gt", float("inf"))], [("f64", "lt", float("-inf"))],
             [("f32", "ge", 5e-324), ("f32", "lt", 1.2e-38)], [("f32", "gt", 0.1), ("f64", "lt", 0.1)]]
    for preds in cases:
        r.check_scan(preds, nan_columns=True)
        r.check_aggregate(preds, AGG_KW, fused=False, nan_columns=True)
        r.check_aggregate(preds, dict(AGG_KW, mode=HG_AGG_HASH), fused=False, nan_columns=True)


# ------------------------------------------------------------------------------- min / max / sum with special values
NAN, NEG_NAN, PAY_NAN = 0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000012345
PZ, NZ, PINF, NINF = 0, 1 << 63, 0x7FF0000000000000, 0xFFF0000000000000
ONE, MONE, TWO, FIVE = bits_of(1.0), bits_of(-1.0), bits_of(2.0), bits_of(5.0)
SPECIAL_VALUES = [NAN, NEG_NAN, PZ, NZ, PINF, NINF, MONE, ONE, TWO]
SERIES, POINTS, DELTA = 64, 512, 1000
W_SLICES = 128 * DELTA             # buckets of 4 slices: the first slice of a bucket opens its group, the others take the fast path


def _special_values_table(nulls):
    """64 series x 512 points (every series starts a slice: lane = point % 32).  Targeted series first, then a seeded mix."""
    rng = np.random.default_rng(17)
    v = [[ONE] * POINTS for _ in range(SERIES)]
    v[0][0] = NAN; v[0][40] = MONE; v[0][77] = PINF                          # a NaN as the group's first value
    v[1][32 + 8] = NAN; v[1][32 + 24] = MONE                                # NaN in lane 8 hides the only minimum in lane 24
    v[2][32 + 8] = NAN; v[2][32 + 24] = FIVE                                # ... and the only maximum
    v[3][160 + 8] = NAN; v[3][160 + 24] = MONE                              # the same in a later bucket's fast-path slice
    for s, first, second in ((4, NZ, PZ), (5, PZ, NZ)):                      # zeros after a first slice of 1.0, lane 0 = 1.0
        for sl in range(1, POINTS // 32):
            v[s][sl * 32 + 8] = first; v[s][sl * 32 + 16] = second
    for s, first, second in ((6, NZ, PZ), (7, PZ, NZ)):                      # max over zeros after a first slice of -1.0
        v[s] = [MONE] * POINTS
        for sl in range(1, POINTS // 32):
            v[s][sl * 32 + 8] = first; v[s][sl * 32 + 16] = second
    v[8] = [ONE] * 32 + [NZ] + [ONE] * 31 + [PZ] * 32 + [ONE] * (POINTS - 96)   # ties across slices: the earlier zero stays
    v[9] = [ONE] * 32 + [PZ] + [ONE] * 31 + [NZ] * 32 + [ONE] * (POINTS - 96)
    v[10] = [[NAN, NEG_NAN, PAY_NAN][i % 3] for i in range(POINTS)]        # all NaN
    v[11] = [PINF if i % 2 else NINF for i in range(POINTS)]                 # inf + -inf in the sum
    v[12] = [NEG_NAN] + [TWO] * (POINTS - 1)
    for s in range(13, SERIES):
        v[s] = [SPECIAL_VALUES[i] for i in rng.integers(0, len(SPECIAL_VALUES), POINTS)]
        v[s][0] = [ONE, PZ, NZ, NAN][s % 4]
    if nulls:
        v[14] = [None] * POINTS                                              # a group whose values are all NULL
        for i in rng.integers(0, POINTS, 60):
            v[15][int(i)] = None
        v[16][0] = None
        v[16][1] = NAN
    user = pa.schema([pa.field("k", pa.uint64(), True), pa.field("t", pa.int64(), True), pa.field("v", pa.float64(), True),
                      pa.field("tag", pa.uint32(), True)])
    cols = {"k": [s for s in range(SERIES) for _ in range(POINTS)],
            "t": [W_SLICES * 10 + i * DELTA for _ in range(SERIES) for i in range(POINTS)],
            "v": [x for s in v for x in s],
            "tag": rng.integers(0, 8, SERIES * POINTS).tolist()}
    return Table(user, cols)


SPECIAL_PREDS = [[], [("tag", "eq", 3)], [("tag", "le", 6)], [("t", "ge", W_SLICES * 10 + 100 * DELTA), ("tag", "ne", 5)],
                 [("t", "ge", W_SLICES * 10 + 33 * DELTA)]]
SPECIAL_KWS = [AGG_KW, dict(group_col=0, ts_col=1, window_ms=W_SLICES, value_col=2), dict(group_col=0, ts_col=1, window_ms=60_000, value_col=2)]


@pytest.fixture(scope="module")
def special_runner():
    t = _special_values_table(nulls=False)
    r = Runner(t, [t.write(4096)])
    yield r
    r.close()


@pytest.mark.parametrize("preds", SPECIAL_PREDS, ids=["all", "sparse", "dense", "ne", "range"])
def test_min_max_sum_special_values(special_runner, preds):
    """NaNs (first value of a group, hiding a minimum in the warp combine, all-NaN groups), signed-zero ties in both orders and
    across slices, infinities of both signs: per series, per bucket, RUNS and HASH, dense groups (the fused fast path) and
    sparse survivors (its per-survivor path).  `!=` takes the general pipeline."""
    fused = not any(op == "ne" for _, op, _ in preds)
    for kw in SPECIAL_KWS:
        special_runner.check_aggregate(preds, kw, fused=fused)


def test_min_max_sum_with_nulls():
    """The same values with NULLs (a group without any value: count only, sum 0.0, min +inf, max -inf): the general pipeline."""
    t = _special_values_table(nulls=True)
    r = Runner(t, [t.write(4096)])
    try:
        for preds in SPECIAL_PREDS[:3]:
            for kw in SPECIAL_KWS[:2]:
                r.check_aggregate(preds, kw, fused=False)
                r.eng.set_flags(0)
                r._agg(0, True, preds, kw)
                assert r.eng.stats()["path"] == 0                    # a nullable value column: the fused planner declines
    finally:
        r.close()


# ------------------------------------------------------------------------------------- timestamps at the ends of i64
@pytest.fixture(scope="module")
def ts_runner():
    rng = np.random.default_rng(23)
    offs = sorted(set(range(0, 40)) | set(rng.integers(0, 200_000, 150).tolist()))
    near = {0: [I64_MIN + o for o in offs], 1: sorted(set(rng.integers(-2500, 2500, 190).tolist()) | {-1, 0, 1}),
            2: [I64_MAX - o for o in reversed(offs)]}
    k, t = [], []
    for s, ts in near.items():
        k += [s] * len(ts)
        t += ts
    user = pa.schema([pa.field("k", pa.uint64(), True), pa.field("t", pa.int64(), True), pa.field("v", pa.float64(), True)])
    tab = Table(user, {"k": k, "t": t, "v": [bits_of(float(x)) for x in rng.integers(-100, 100, len(k)) / 4]})
    r = Runner(tab, [tab.write(8192)])
    yield r
    r.close()


@pytest.mark.parametrize("w", [1, 7, 1000, 60_000, I64_MAX])
def test_buckets_at_the_ends_of_i64(ts_runner, w):
    """Rows within a few windows of i64 min and of i64 max (and around 0, where the bucket spans 2w - 1): bucket starts by
    truncating division, on every aggregate path."""
    kw = dict(group_col=0, ts_col=1, window_ms=w, value_col=2)
    for preds in ([], [("t", "ge", I64_MIN + 3), ("t", "le", I64_MAX - 2)], [("t", "lt", I64_MIN + 1)], [("t", "gt", I64_MAX - 1)]):
        ts_runner.check_aggregate(preds, kw)
    ts_runner.check_aggregate([("t", "ge", 0), ("t", "lt", 0)], COUNT_KW)
