"""The k-way merge and dedup (S4-S6: SortPreservingMergeExec on (pk.., __seq__), ties to the lower stream, then LastValueOperator /
BytesMergeOperator over the primary-key runs) at the limits of their shape: 63-300 streams, keys at the 52-bit budget of the packed
single pass (kway_merge.cu), every primary-key layout validate_schema allows, __seq__ NULL / tied / at u64 max, and runs that cross
the merge's key ranges and rounds.

Every call goes through the C ABI twice, with the packed pass allowed and under HG_FLAG_PAIRWISE_MERGE (the merge-path passes of
kernels.cu): both outputs must be identical, and the launch counts must show which path ran (the packed pass launches 5 kernels, the
pairwise passes 3 + 2 * ceil(log2 k)).  Which path is expected comes from `Table.packed`, a restatement of plan_key_pack's rule:
k <= 128 streams and (pk.., __seq__ + 1, stream) within 52 bits after rebasing every field to the statistics.  Each result is
compared with the oracle (rows, bytes, validity and MergeStream batch boundaries) and with `Table.expected`, a numpy model of the
merge written here: filter each file, stable-sort all rows by (pk.., __seq__ NULLS FIRST, stream, position in the file), keep the
last row of every primary-key run."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from horaedb_b200 import sstgen
from horaedb_b200._ffi import HG_AGG_HASH, HG_AGG_RUNS, HG_FLAG_PAIRWISE_MERGE, Engine, HgError, SchemaHandle, SstInput
from horaedb_b200.config import WriteConfig
from horaedb_b200.types import StorageSchema, UpdateMode
from oracle import oracle
from oracle.merge_stream import BytesMergeOperator, MergeStream

from helpers import arrays_equal, arrow_schema, check_stream

pytestmark = pytest.mark.gpu
_next_id = iter(range(120_000_000, 130_000_000))
_NP = {"uint8": np.uint8, "int8": np.int8, "uint32": np.uint32, "int32": np.int32, "uint64": np.uint64, "int64": np.int64}
_CODECS = ("snappy", "none", "zstd")
_ROW_GROUPS = (8192, 5, 64)
U64_MAX = (1 << 64) - 1
T0 = sstgen.T0_MS


class Table:
    """A table's storage schema, its SSTs in stream order, and the rows each SST holds (numpy, in file order).  Value columns:
    `w` = the file's index (int32), `v` = a float64 derived from `rid`, `rid` = a row id that grows in stream order and file
    order; an Append-mode table has one Binary column `blob` instead (`rid` is then kept for the model only)."""

    def __init__(self, pk_spec, mode=UpdateMode.Overwrite):
        self.pk = [n for n, _ in pk_spec]
        self.append = mode == UpdateMode.Append
        values = [("blob", "binary")] if self.append else [("w", "int32"), ("v", "float64"), ("rid", "uint64")]
        self.user = arrow_schema(list(pk_spec) + values)
        self.schema = StorageSchema.try_new(self.user, len(pk_spec), mode)
        self.handle = SchemaHandle(self.schema.arrow_schema, len(pk_spec), mode)
        self.types = {n: t for n, t in pk_spec}
        self.files, self.datas = [], []
        self.rid = 0

    def add(self, pks, seq, seq_valid=None, codec="snappy", rg=8192):
        """One SST with the rows `pks` (one array per PK column), sorted by (pk.., __seq__ NULLS FIRST) as a file is; `seq` a scalar
        or one value per row; `seq_valid` False where __seq__ is NULL.  Rows equal in both keep their given order."""
        n = len(pks[0])
        cols = {name: np.asarray(a, dtype=_NP[self.types[name]]) for name, a in zip(self.pk, pks)}
        valid = np.ones(n, bool) if seq_valid is None else np.asarray(seq_valid, bool)
        seq = np.where(valid, np.broadcast_to(np.asarray(seq, dtype=np.uint64), (n,)), np.uint64(0))
        order = np.lexsort([seq, valid] + [cols[c] for c in reversed(self.pk)])
        cols = {c: a[order] for c, a in cols.items()}
        cols["__seq__"], cols["_valid"] = seq[order], valid[order]
        cols["rid"] = np.arange(self.rid, self.rid + n, dtype=np.uint64)
        self.rid += n
        f = len(self.files)
        cols["w"] = np.full(n, f, np.int32)
        cols["v"] = (sstgen.splitmix64(cols["rid"]) >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53))
        if self.append:
            cols["blob"] = np.array([b"%d." % r * (1 + r % 3) for r in cols["rid"].tolist()], dtype=object)
        arrays = [pa.array(cols[fl.name].tolist() if fl.type == pa.binary() else cols[fl.name], fl.type) for fl in self.user]
        arrays += [pa.array(cols["__seq__"], pa.uint64(), mask=~cols["_valid"]), pa.nulls(n, pa.uint64())]
        batch = pa.RecordBatch.from_arrays(arrays, schema=self.schema.arrow_schema)
        self.datas.append(sstgen.write_sst_with_seq(self.schema, batch, WriteConfig(compression=codec, max_row_group_size=rg)))
        self.files.append(cols)

    @property
    def k(self):
        return len(self.files)

    def key_bits(self):
        """plan_key_pack's budget: ceil(log2 k) stream bits + the bits of the __seq__ + 1 span (NULL = 0, so a NULL makes the span
        start at 0) + the bits of every PK column's span, over the statistics of every file.  None when __seq__ reaches u64 max."""
        rows = [f for f in self.files if len(f["rid"])]
        seq = np.concatenate([f["__seq__"][f["_valid"]] for f in rows])
        nullable = any(not f["_valid"].all() for f in rows)
        if len(seq) == 0:
            seq_span = 0
        else:
            lo, hi = int(seq.min()), int(seq.max())
            if hi == U64_MAX:
                return None
            seq_span = hi + 1 - (0 if nullable else lo + 1)
        used = (self.k - 1).bit_length() + seq_span.bit_length()
        for c in self.pk:
            a = np.concatenate([f[c] for f in rows])
            used += (int(a.max()) - int(a.min())).bit_length()
        return used

    def packed(self):
        bits = self.key_bits()
        return self.k <= 128 and bits is not None and bits <= 52

    def merged(self, preds=()):
        """Every row that passes `preds`, in merge order: (pk.., __seq__ NULLS FIRST, stream, position)."""
        parts = [{c: a[_mask(f, preds)] for c, a in f.items()} for f in self.files]
        cat = {c: np.concatenate([p[c] for p in parts]) for c in parts[0]}
        order = np.lexsort([cat["rid"], cat["__seq__"], cat["_valid"]] + [cat[c] for c in reversed(self.pk)])
        return {c: a[order] for c, a in cat.items()}

    def expected(self, preds=()):
        """LastValueOperator: the last row of every primary-key run of the merged rows."""
        m = self.merged(preds)
        n = len(m["rid"])
        last = np.ones(n, bool)
        if n:
            last[:-1] = np.logical_or.reduce([m[c][1:] != m[c][:-1] for c in self.pk])
        return {c: a[last] for c, a in m.items()}

    def expected_append(self, keep_builtin, batch_size=8192):
        """BytesMergeOperator through oracle/merge_stream.py, fed the merged rows in batches of `batch_size`."""
        m = self.merged()
        tbl = pa.table({fl.name: _arrow(m, fl, len(m["rid"])) for fl in self.schema.arrow_schema}, schema=self.schema.arrow_schema)
        batches = [tbl.slice(lo, batch_size).combine_chunks().to_batches()[0] for lo in range(0, tbl.num_rows, batch_size)]
        return list(MergeStream(batches, len(self.pk), BytesMergeOperator(self.schema.value_idxes), keep_builtin))

    def inputs(self, resident=()):
        return [SstInput(id=resident[i]) if i in resident else SstInput(id=next(_next_id), data=d) for i, d in enumerate(self.datas)]


_OPS = {"eq": np.equal, "ne": np.not_equal, "lt": np.less, "le": np.less_equal, "gt": np.greater, "ge": np.greater_equal}


def _mask(cols, preds):
    m = np.ones(len(cols["rid"]), bool)
    for c, op, lit in preds:
        m &= np.isin(cols[c], lit) if op == "in" else _OPS[op](cols[c], lit)
    return m


def _arrow(rows, field, n):
    if field.name == "__seq__":
        return pa.array(rows["__seq__"], pa.uint64(), mask=~rows["_valid"])
    if field.name == "__reserved__":
        return pa.nulls(n, pa.uint64())
    return pa.array(rows[field.name].tolist() if field.type == pa.binary() else rows[field.name], field.type)


def _check_rows(t, got, rows):
    """`got` (batches or a table) holds exactly the model's rows, column by column (values and validity)."""
    n = len(rows["rid"])
    if not isinstance(got, pa.Table) and not got:
        assert n == 0, f"no rows, the model keeps {n}"
        return
    tbl = got if isinstance(got, pa.Table) else pa.Table.from_batches(got)
    assert tbl.num_rows == n, f"{tbl.num_rows} rows, the model keeps {n}"
    for name in tbl.column_names:
        exp = _arrow(rows, t.schema.arrow_schema.field(name), n)
        if not arrays_equal(tbl[name], exp):
            a, e = tbl[name].to_pylist(), exp.to_pylist()
            bad = [i for i in range(n) if a[i] != e[i]]
            raise AssertionError(f"column {name}: {len(bad)} of {n} rows differ from the model, first {[(i, a[i], e[i]) for i in bad[:4]]}")


def _both_paths(eng, t, call, compare=check_stream):
    """`call()` with the packed single pass allowed, then under HG_FLAG_PAIRWISE_MERGE.  The two results must be identical, and the
    launch counts must name the path the first call took: the pairwise passes launch 2 * ceil(log2 k) - 2 more kernels (k >= 3)."""
    assert t.k >= 3, "at k = 2 both paths launch 5 kernels"
    out, launches = [], []
    for flags in (0, HG_FLAG_PAIRWISE_MERGE):
        eng.set_flags(flags)
        out.append(call())
        launches.append(eng.stats()["kernel_launches"])
    eng.set_flags(0)
    packed = t.packed()
    extra = 2 * (t.k - 1).bit_length() - 2 if packed else 0
    assert launches[1] - launches[0] == extra, (f"k = {t.k}, key bits {t.key_bits()}: expected the {'packed' if packed else 'pairwise'} "
                                                f"path, launches {launches[0]} (flags 0) vs {launches[1]} (pairwise)")
    compare(out[1], out[0])
    return out[0]


def _scan(eng, t, preds=(), keep_builtin=True, batch_size=8192, resident=()):
    """One scan on both paths, checked against the oracle and the model."""
    got = _both_paths(eng, t, lambda: list(eng.scan(t.handle, t.inputs(resident), preds, None, keep_builtin)))
    check_stream(got, oracle.scan(t.datas, t.schema.arrow_schema, len(t.pk), preds, keep_builtin, batch_size).batches)
    _check_rows(t, got, t.expected(preds))
    return got


def _universe(rng, n, sids=40, points=30):
    """`n` distinct (series_id, ts) keys of a `sids` x `points` grid, sorted."""
    pick = np.sort(rng.choice(sids * points, size=min(n, sids * points), replace=False))
    return [(pick // points).astype(np.uint64), T0 + (pick % points).astype(np.int64) * 1000]


_METRIC_PK = [("series_id", "uint64"), ("ts", "int64")]


# ------------------------------------------------------------------------------------------------------------ stream counts
@pytest.mark.parametrize("k", [63, 64, 65, 100, 127, 128, 129, 200, 300])
def test_stream_counts(k):
    """k small, heavily overlapping files (every PK in several of them, some files empty), codec and row-group size varying per
    file, __seq__ a permutation of the file order; 65-128 streams take B = 32 keys per stream per round and a 7-level tree with k
    padded to pairs, more than 128 the pairwise passes.  Then predicates that leave 2 or 3 streams, and one that thins every stream."""
    rng = np.random.default_rng(k)
    t = Table(_METRIC_PK)
    seqs = 1000 + rng.permutation(k)
    for f in range(k):
        n = 0 if f % 23 == 5 else int(rng.integers(20, 150))
        t.add(_universe(rng, n), seqs[f], codec=_CODECS[f % 3], rg=_ROW_GROUPS[f % 3])
    assert t.packed() == (k <= 128)
    few = [f for f in range(k) if len(t.files[f]["rid"])]
    eng = Engine(device=0)
    for preds, keep_builtin, streams in (((), True, None), ([("w", "in", [few[1], few[k // 2], few[-1]])], False, 3),
                                         ([("w", "ge", few[-2])], True, 2), ([("v", "lt", 0.3)], False, None)):
        got = _scan(eng, t, preds, keep_builtin)
        if streams:
            assert len(set(t.merged(preds)["w"].tolist())) == streams
            assert 0 < pa.Table.from_batches(got).num_rows < len(t.merged(preds)["w"])
    eng.close()


# ------------------------------------------------------------------------------------------------------ the 52-bit boundary
@pytest.mark.parametrize("k", [3, 128])
@pytest.mark.parametrize("bits", [52, 53])
def test_packed_key_budget_boundary(k, bits):
    """PK statistics chosen so that (pk0 i64 crossing zero, pk1 u32 spanning 8 bits, __seq__ + 1, stream) need exactly 52 bits
    (packed single pass) or 53 (pairwise passes), at k = 3 (2 stream bits) and k = 128 (7)."""
    rng = np.random.default_rng(bits * 1000 + k)
    t = Table([("a", "int64"), ("b", "uint32")])
    rb = (k - 1).bit_length()
    seqs = 10 + np.arange(k) % 3 if k == 3 else 1000 + rng.permutation(k)           # __seq__ + 1 spans 2 bits (k = 3), 7 (k = 128)
    sb = (int(seqs.max()) - int(seqs.min())).bit_length()
    a_span = (1 << (bits - rb - sb - 8)) - 1                                       # b spans 255: 8 bits
    a_lo = -(a_span // 2) - 3
    a_vals = np.unique(np.concatenate([[a_lo, a_lo + a_span, -1, 0], a_lo + rng.integers(0, a_span + 1, 40)]))
    b_vals = np.unique(np.concatenate([[0, 255], rng.integers(0, 256, 10)]))
    grid = np.array([(x, y) for x in a_vals for y in b_vals], dtype=object)
    for f in range(k):
        rows = grid[np.sort(rng.choice(len(grid), size=60 if k == 3 else 12, replace=False))]
        if f < 2:                                                                  # the extremes are in the statistics
            rows = np.concatenate([rows, [(a_lo, 0), (a_lo + a_span, 255)]])
        t.add([[int(x) for x in rows[:, 0]], [int(y) for y in rows[:, 1]]], int(seqs[f]), codec=_CODECS[f % 3], rg=_ROW_GROUPS[f % 3])
    assert t.key_bits() == bits and t.packed() == (bits == 52)
    eng = Engine(device=0)
    _scan(eng, t)
    _scan(eng, t, [("v", "ge", 0.5)], keep_builtin=False)
    eng.close()


@pytest.mark.parametrize("top", [U64_MAX - 1, U64_MAX])
def test_seq_at_the_top_of_u64(top):
    """__seq__ at u64 max - 1 (its value + 1 still fits: packed when the span is small) and at u64 max (value + 1 does not: always
    the pairwise passes).  Files 0 and 3 tie at the top, so the higher stream wins; a second table adds files with a small __seq__."""
    rng = np.random.default_rng(top & 7)
    eng = Engine(device=0)
    for seqs in ([top, top - 1, top - 2, top], [top, 3, top - 1, top, 7]):
        t = Table([("k", "uint64")])
        for f, s in enumerate(seqs):
            t.add([np.sort(rng.choice(400, 150, replace=False)).astype(np.uint64) + np.uint64(1 << 63)], s, codec=_CODECS[f % 3], rg=_ROW_GROUPS[f % 3])
        assert t.packed() == (top < U64_MAX and seqs[1] > 3)
        got = pa.Table.from_batches(_scan(eng, t))
        key, seq, w = got["k"].to_numpy(), got["__seq__"].to_numpy(), got["w"].to_numpy()
        in0, in3 = np.isin(key, t.files[0]["k"]), np.isin(key, t.files[3]["k"])
        assert in3.any() and (in0 & ~in3).any()
        assert (seq[in0 | in3] == top).all() and (w[in3] == 3).all() and (w[in0 & ~in3] == 0).all()
    eng.close()


# ---------------------------------------------------------------------------------------------------------- PK layouts
def _type_values(t, width, c, rng):
    info = np.iinfo(_NP[t])
    lo, hi = int(info.min), int(info.max)
    if width == "full":
        edges = np.array([lo, lo + 1, max(lo, -1), 0, 1, hi - 1, hi], dtype=_NP[t])
        return np.unique(np.concatenate([edges, rng.integers(lo, hi, 3, dtype=_NP[t], endpoint=True)]))
    if lo < 0:
        base = lo if c % 2 == 0 else hi - 7                      # at the bottom or the top of a signed type
    else:
        base = (hi + 1) // 2 - 3 if c % 2 == 0 else hi - 7      # across the sign bit of the same-width signed type, or at the top
    return np.array([base + i for i in range(8)], dtype=_NP[t])


@pytest.mark.parametrize("width", ["narrow", "full"])
@pytest.mark.parametrize("layout", [("int8",), ("uint64", "uint64"), ("uint32", "int32"), ("int32", "uint8", "int64"),
                                    ("int8", "uint8", "uint32", "int64"), ("int64", "uint64")])
def test_primary_key_layouts(layout, width):
    """1-4 PK columns (u64 + u64: exactly 16 bytes) with values at the type extremes (i8 -128 / 127, i32 and i64 min / max, u64 at and
    above 2^63): "narrow" keeps every column within 8 values of an extreme, so the key packs after rebasing; "full" spans every type's
    whole range, so the wide layouts take the pairwise passes."""
    rng = np.random.default_rng(len(layout) * 10 + (width == "full"))
    t = Table([(f"p{c}", ty) for c, ty in enumerate(layout)])
    vals = [_type_values(ty, width, c, rng) for c, ty in enumerate(layout)]
    grid = np.stack([g.ravel() for g in np.meshgrid(*[np.arange(len(v)) for v in vals], indexing="ij")], axis=1)
    for f in range(6):
        sel = grid[np.sort(rng.choice(len(grid), size=min(len(grid), 90), replace=False))]
        if f == 0:
            sel = np.concatenate([sel, [[0] * len(layout), [len(v) - 1 for v in vals]]])
        t.add([vals[c][sel[:, c]] for c in range(len(layout))], [50, 51, 50, 53, 52, 53][f], codec=_CODECS[f % 3], rg=_ROW_GROUPS[f % 3])
    assert t.packed() == (width == "narrow" or layout == ("int8",))
    eng = Engine(device=0)
    _scan(eng, t)
    _scan(eng, t, [("p0", "ne", int(vals[0][1]))], keep_builtin=False)
    eng.close()


def test_seventeen_byte_primary_key_is_refused():
    user = arrow_schema([("a", "uint64"), ("b", "uint64"), ("c", "uint8"), ("v", "float64")])
    schema = StorageSchema.try_new(user, 3)
    data = sstgen.write_sst(schema, pa.RecordBatch.from_pydict({"a": [1], "b": [2], "c": [3], "v": [0.5]}, schema=user), seq=1)
    eng = Engine(device=0)
    for call in (lambda h: eng.scan(h, [SstInput(id=next(_next_id), data=data)] * 3), lambda h: eng.compact(h, [SstInput(id=next(_next_id), data=data)])):
        with pytest.raises(HgError) as ei:
            call(SchemaHandle(schema.arrow_schema, 3))
        assert ei.value.code == 2 and "wider than 128 bits" in str(ei.value)
    eng.close()


# ------------------------------------------------------------------------------------------------------------ __seq__ domain
@pytest.mark.parametrize("k", [6, 130])
def test_seq_nulls_ties_and_intra_file_duplicates(k):
    """Per file, by index mod 6: every __seq__ NULL, some NULL, 77 as in the next file (ties: the higher stream wins), 77 with
    intra-file duplicates of identical (pk, __seq__) (the later row in the file wins), distinct and lower.  k = 6 packs with __seq__
    rebased to 0 (the NULL domain), k = 130 takes the pairwise passes."""
    rng = np.random.default_rng(k)
    t = Table([("a", "int32"), ("b", "uint8")])
    keys = np.array([(a, b) for a in range(-20, 20) for b in (0, 7, 255)])
    for f in range(k):
        rows = keys[np.sort(rng.choice(len(keys), size=40, replace=False))]
        kind, valid, seq = f % 6, None, 77
        if kind == 0:
            valid = np.zeros(len(rows), bool)
        elif kind == 1:
            valid, seq = rng.random(len(rows)) < 0.6, rng.choice([5, 40, 77], len(rows))
        elif kind == 4:
            rows = np.repeat(rows, rng.integers(1, 4, len(rows)), axis=0)
        elif kind == 5:
            seq = 10 + f % 60
        t.add([rows[:, 0], rows[:, 1]], seq, valid, codec=_CODECS[f % 3], rg=_ROW_GROUPS[(f // 3) % 3])
    assert t.packed() == (k <= 128)
    # runs whose winner ties with the row before it in (pk, __seq__): from a higher stream, and from the same file
    m = t.merged()
    same_pk = (m["a"][1:] == m["a"][:-1]) & (m["b"][1:] == m["b"][:-1])
    won_by_tie = same_pk & (m["__seq__"][1:] == m["__seq__"][:-1]) & m["_valid"][1:] & m["_valid"][:-1] & np.append(~same_pk[1:], True)
    assert (won_by_tie & (m["w"][1:] > m["w"][:-1])).sum() > 5 and (won_by_tie & (m["w"][1:] == m["w"][:-1])).sum() > 5
    eng = Engine(device=0)
    _scan(eng, t)
    _scan(eng, t, [("b", "eq", 7)], keep_builtin=False)
    eng.close()


# ---------------------------------------------------------------------------------------------------------- ranges and rounds
def _runs_table(k, npks, frac, hot, seed):
    """k files over one set of `npks` PKs, each PK in a `frac` share of them; one hot PK in every file with `hot` versions in all,
    repeated inside each file with the file's __seq__; files share __seq__ values in pairs."""
    rng = np.random.default_rng(seed)
    t = Table(_METRIC_PK)
    sid = np.arange(npks, dtype=np.uint64) // 50
    ts = T0 + (np.arange(npks, dtype=np.int64) % 50) * 1000
    h = npks // 2
    seqs = 1000 + rng.permutation(k) // 2
    for f in range(k):
        keep = rng.random(npks) < frac
        reps = np.ones(npks, np.int64)
        reps[h] = hot // k
        keep[h] = True
        idx = np.repeat(np.flatnonzero(keep), reps[keep])
        t.add([sid[idx], ts[idx]], seqs[f], codec=_CODECS[f % 3], rg=(8192, 1000, 65536)[f % 3])
    return t, (sid[h], ts[h])


def _check_runs(t, hot):
    n = sum(len(f["rid"]) for f in t.files)
    versions = sum(int(((f["series_id"] == hot[0]) & (f["ts"] == hot[1])).sum()) for f in t.files)
    assert n // 16384 >= 6 and versions > 16384 and t.packed()       # 6+ key ranges of 16384 rows; one PK run longer than a range
    eng = Engine(device=0)
    _scan(eng, t)
    eng.close()


def test_pk_runs_across_ranges_and_rounds():
    """~120 000 rows in 100 files: 7 key ranges of the packed pass, rounds of 32 keys per stream, every PK in most files (runs of
    ~80 versions cross round ends and range cuts) and one PK with 24 000 versions, 240 per file as intra-file duplicates."""
    _check_runs(*_runs_table(100, 1200, 0.8, 24_000, 1))


def test_pk_runs_across_ranges_and_rounds_large():
    """The same shape at 3.2 M rows: hundreds of key ranges."""
    _check_runs(*_runs_table(100, 40_000, 0.8, 30_000, 2))


# ------------------------------------------------------------------------------------------------------------ entry points
def _entry_table(k, mode=UpdateMode.Overwrite):
    rng = np.random.default_rng(k + mode)
    t = Table([("series_id", "uint64"), ("ts", "int64")] if mode == UpdateMode.Overwrite else [("a", "uint64"), ("b", "int8")], mode)
    seqs = 2000 + rng.permutation(k)
    for f in range(k):
        u = _universe(rng, 0 if f % 31 == 7 else int(rng.integers(30, 60)), sids=30, points=20)
        if mode == UpdateMode.Append:
            u = [u[0], (u[1] - T0) // 1000 - 10]
        t.add(u, seqs[f], codec=_CODECS[f % 3], rg=_ROW_GROUPS[f % 3])
    return t


def _load_half(eng, t):
    ids = {}
    for i in range(0, t.k, 2):
        ids[i] = next(_next_id)
        eng.load_sst(t.handle, SstInput(id=ids[i], data=t.datas[i]))
    return ids


@pytest.mark.parametrize("k", [128, 129])
def test_scan_entry_points_at_the_stream_limit(k):
    """scan with and without the builtin columns at batch sizes 1, 7 and 8192 (MergeStream's boundaries), with every SST transient and
    with resident and transient SSTs mixed in one call."""
    t = _entry_table(k)
    for bs in (1, 7, 8192):
        eng = Engine(device=0, batch_size=bs)
        resident = _load_half(eng, t)
        for keep_builtin in (True, False):
            for res in ((), resident):
                _scan(eng, t, (), keep_builtin, bs, res)
        eng.close()


def _check_agg(got, want, gname):
    assert got.num_rows == len(want["count"])
    assert got[gname].to_pylist() == list(want["group"]) and got["count"].to_pylist() == list(want["count"])
    for c in ("sum", "min", "max"):
        assert np.array_equal(got[c].to_numpy().view(np.uint64), np.asarray(want[c], np.float64).view(np.uint64)), c


def _model_agg(rows, key):
    """count / sum (sequential f64 adds in stream order) / min / max per group of `key`, groups sorted by key."""
    acc = {}
    for g, x in zip(rows[key].tolist(), rows["v"].tolist()):
        c, s, lo, hi = acc.get(g, (0, 0.0, x, x))
        acc[g] = (c + 1, s + x, min(lo, x), max(hi, x))
    gs = sorted(acc)
    return {"group": gs, "count": [acc[g][0] for g in gs], "sum": [acc[g][1] for g in gs], "min": [acc[g][2] for g in gs],
            "max": [acc[g][3] for g in gs]}


def _tables_equal(a, b):
    assert a.schema.names == b.schema.names and a.num_rows == b.num_rows
    for c in a.column_names:
        assert arrays_equal(a[c], b[c]), c


@pytest.mark.parametrize("k", [128, 129])
def test_compaction_and_aggregates_at_the_stream_limit(k, tmp_path):
    """hg_compact_open, hg_compact_to_sst (read back with pyarrow) and RUNS / HASH aggregates after dedup (f64 sums bit for bit against
    the oracle and against sequential sums over the model's rows), resident and transient SSTs mixed."""
    t = _entry_table(k)
    eng = Engine(device=0)
    res = _load_half(eng, t)
    rows = t.expected()
    got = _both_paths(eng, t, lambda: list(eng.compact(t.handle, t.inputs(res))))
    check_stream(got, oracle.scan(t.datas, t.schema.arrow_schema, 2, (), True, 8192).batches)
    _check_rows(t, got, rows)
    paths = iter(range(2))

    def to_sst():
        path = str(tmp_path / f"out{next(paths)}.sst")
        eng.compact_to_sst(t.handle, t.inputs(res), path, max_row_group_size=1000)
        return pq.read_table(path)

    _check_rows(t, _both_paths(eng, t, to_sst, _tables_equal), rows)
    v = t.schema.arrow_schema.get_field_index("v")
    w = t.schema.arrow_schema.get_field_index("w")
    for mode, kw, gname, key in ((HG_AGG_RUNS, dict(group_col=0, ts_col=-1, window_ms=0), "series_id", "series_id"),
                                 (HG_AGG_RUNS, dict(group_col=0, ts_col=1, window_ms=5000), "series_id", None),
                                 (HG_AGG_HASH, dict(group_col=w, ts_col=-1, window_ms=0), "w", "w")):
        got = _both_paths(eng, t, lambda: eng.scan_aggregate(t.handle, t.inputs(res), [], value_col=v, mode=mode, **kw), _tables_equal)
        exp = oracle.scan_aggregate(t.datas, t.schema.arrow_schema, 2, [], value_col=v, mode=mode, **kw)
        _check_agg(got, {"group": exp.gkey.astype(np.int64 if gname == "w" else np.uint64).tolist(), "count": exp.count.tolist(), "sum": exp.sum,
                         "min": exp.min, "max": exp.max}, gname)
        if key:
            _check_agg(got, _model_agg(rows, key), gname)
        else:
            assert got["bucket"].to_pylist() == exp.bucket.tolist()
    eng.close()


@pytest.mark.parametrize("k", [128, 129])
def test_append_mode_binary_values_at_the_stream_limit(k):
    """UpdateMode::Append with a Binary value column: BytesMergeOperator concatenates each run's bytes in merge order, against
    oracle/merge_stream.py fed the model's merged rows; resident and transient SSTs mixed."""
    t = _entry_table(k, UpdateMode.Append)
    eng = Engine(device=0)
    res = _load_half(eng, t)
    for keep_builtin in (True, False):
        for r in ((), res):
            got = _both_paths(eng, t, lambda: list(eng.scan(t.handle, t.inputs(r), (), None, keep_builtin)))
            exp = t.expected_append(keep_builtin)
            assert len(got) == len(exp)
            for a, e in zip(got, exp):
                assert a.schema.names == e.schema.names and a.num_rows == e.num_rows
                for c in range(a.num_columns):
                    assert arrays_equal(a.column(c), e.column(c)), a.schema.names[c]
    eng.close()
