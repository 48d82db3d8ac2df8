"""TEST INFRASTRUCTURE: the model of the aggregates by label group (`hg_scan_aggregate_by_map`, `hg_scan_quantile_aggregate_by_map`).  A
plain Python restatement over the deduplicated stream of the C oracle (`oracle.scan`); it uses nothing of the library.

A row whose key is not in the map (or is NULL) does not take part.  Every other row belongs to (map[key], bucket); a group's count is its
rows, its sum the f64 sum of its non-NULL values added one by one in stream order (Python floats round every addition, as the device
does), its min / max those of reduce_groups (the first value, then `v < min` / `v > max`: a NaN only when it comes first; +inf / -inf
without a value).  Groups are sorted by (ordinal, bucket).  Quantiles reuse `quantile_model.quantiles_of`."""
from __future__ import annotations

import numpy as np
import pyarrow as pa

from oracle import oracle
from quantile_model import _trunc_div, quantiles_of

INF = float("inf")


def map_lookup(key_t: pa.DataType, keys, groups):
    """{key as the column's Python value: ordinal} of a map given in the widened domain (i64 / u64 two's complement).  A key the
    column cannot hold stays in the dict and never matches a row; a key given twice must repeat its group."""
    out = {}
    signed = pa.types.is_signed_integer(key_t)
    ks = keys.astype(np.uint64).tolist() if isinstance(keys, np.ndarray) else [int(k) & 0xFFFFFFFFFFFFFFFF for k in keys]
    for k, g in zip(ks, np.asarray(groups).astype(np.uint64).tolist()):
        v = k - (1 << 64) if signed and k >= 1 << 63 else k
        assert out.setdefault(v, g) == g, "a key mapped to two groups"
    return out


def grouped_rows(ssts, schema: pa.Schema, num_pk: int, preds, group_col: int, keys, groups, ts_col: int = -1, window_ms: int = 0,
                 value_col: int = -1):
    """[(ordinal, bucket, count, [non-NULL values in stream order])] sorted by (ordinal, bucket)"""
    lookup = map_lookup(schema.field(group_col).type, keys, groups)
    res = oracle.scan(ssts, schema, num_pk, preds)
    has_ts = ts_col >= 0 and window_ms > 0
    acc = {}
    for b in res.batches:
        n = b.num_rows
        k = b.column(group_col).to_pylist()
        t = b.column(ts_col).to_pylist() if has_ts else [0] * n
        v = b.column(value_col).to_pylist() if value_col >= 0 else [None] * n
        for key, ts, val in zip(k, t, v):
            g = lookup.get(key) if key is not None else None
            if g is None:
                continue
            if has_ts and ts >= 1 << 63:
                ts -= 1 << 64
            bucket = _trunc_div(ts, window_ms) * window_ms if has_ts else 0
            grp = acc.setdefault((g, bucket), [0, []])
            grp[0] += 1
            if val is not None:
                grp[1].append(val)
    return [(g, bk, c, vals) for (g, bk), (c, vals) in sorted(acc.items())]


def sum_min_max(vals):
    s, mn, mx, seen = 0.0, INF, -INF, False
    for x in vals:
        x = float(x)
        s += x
        if not seen or x < mn:
            mn = x
        if not seen or x > mx:
            mx = x
        seen = True
    return s, mn, mx


def _key_cols(rows, has_ts):
    cols = [pa.array([r[0] for r in rows], pa.uint32())]
    names = ["group"]
    if has_ts:
        cols.append(pa.array([r[1] for r in rows], pa.int64()))
        names.append("bucket")
    cols.append(pa.array([r[2] for r in rows], pa.uint64()))
    names.append("count")
    return cols, names


def aggregate_by_map(ssts, schema: pa.Schema, num_pk: int, preds=(), group_col: int = 0, keys=(), groups=(), ts_col: int = -1,
                     window_ms: int = 0, value_col: int = -1) -> pa.Table:
    """The table `Engine.scan_aggregate_by_map` returns for the same arguments (`schema`: the full storage schema)."""
    rows = grouped_rows(ssts, schema, num_pk, preds, group_col, keys, groups, ts_col, window_ms, value_col)
    cols, names = _key_cols(rows, ts_col >= 0 and window_ms > 0)
    if value_col >= 0:
        smm = [sum_min_max(r[3]) for r in rows]
        for j, name in enumerate(("sum", "min", "max")):
            cols.append(pa.array([x[j] for x in smm], pa.float64()))
            names.append(name)
    return pa.Table.from_arrays(cols, names=names)


def quantile_aggregate_by_map(ssts, schema: pa.Schema, num_pk: int, preds=(), group_col: int = 0, keys=(), groups=(), ts_col: int = -1,
                              window_ms: int = 0, value_col: int = 2, quantiles=(0.5,)) -> pa.Table:
    """The table `Engine.scan_quantile_aggregate_by_map` returns for the same arguments."""
    rows = grouped_rows(ssts, schema, num_pk, preds, group_col, keys, groups, ts_col, window_ms, value_col)
    cols, names = _key_cols(rows, ts_col >= 0 and window_ms > 0)
    vt = schema.field(value_col).type
    per = [quantiles_of(r[3], vt, quantiles) for r in rows]
    for j in range(len(quantiles)):
        cols.append(pa.array([p[j] for p in per], pa.float64()))
        names.append("quantile_%d" % j)
    return pa.Table.from_arrays(cols, names=names)


def reduce_shards(shards):
    """The multi-shard definition of a REDUCE combine of by-map partials: shard tables (as aggregate_by_map returns them, with a value
    column) in rank order; counts summed, f64 sums added in rank order, min / max taken.  {(ordinal, bucket): [count, sum, min, max]}"""
    acc = {}
    for t in shards:
        d = t.to_pydict()
        buckets = d.get("bucket", [0] * t.num_rows)
        for i in range(t.num_rows):
            key = (d["group"][i], buckets[i])
            c, s, mn, mx = d["count"][i], d["sum"][i], d["min"][i], d["max"][i]
            if key not in acc:
                acc[key] = [c, s, mn, mx]
            else:
                a = acc[key]
                a[0] += c
                a[1] = a[1] + s
                a[2] = min(a[2], mn)
                a[3] = max(a[3], mx)
    return acc
