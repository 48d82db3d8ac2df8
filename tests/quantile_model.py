"""TEST INFRASTRUCTURE: the model of `hg_scan_quantile_aggregate`.  A plain Python restatement of the quantiles per (group, bucket) over the
deduplicated stream of the C oracle (`oracle.scan`); it uses nothing of the library.

RUNS: a group is a run of consecutive rows with the same (key, bucket).  HASH: all rows with the same (key, bucket), groups ordered by
(the key's order key, bucket).  Within a group the non-NULL values are ordered by their order key (integers numerically, floats in IEEE
totalOrder, computed here from the f64 bits), converted to f64 (Python's float(int) rounds to nearest, as the C conversion does), and
  rank = q * (m - 1), lo = floor(rank), hi = min(lo + 1, m - 1), w = rank - lo,  result = v(lo) if w == 0 else v(lo) * (1 - w) + v(hi) * w
with Python floats, whose operations each round once (CPython never fuses a multiply-add)."""
from __future__ import annotations

import math
import struct

import pyarrow as pa

from oracle import oracle

HG_AGG_HASH = 1


def _trunc_div(a: int, b: int) -> int:
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def order_key(x, t: pa.DataType) -> int:
    """order_key(widen(x)) of device_types.h for a Python value of Arrow type t"""
    if pa.types.is_floating(t):
        bits = struct.unpack("<Q", struct.pack("<d", float(x)))[0]
        return bits ^ ((1 << 64) - 1 if bits >> 63 else 1 << 63)
    if pa.types.is_signed_integer(t):
        return int(x) + (1 << 63)
    return int(x)


def quantiles_of(values, t: pa.DataType, qs):
    """the quantiles of one group's non-NULL values (None for each q when there are none)"""
    m = len(values)
    if m == 0:
        return [None] * len(qs)
    v = [float(x) for x in sorted(values, key=lambda x: order_key(x, t))]
    out = []
    for q in qs:
        rank = q * (m - 1)
        lo = math.floor(rank)
        hi = min(lo + 1, m - 1)
        w = rank - lo
        out.append(v[lo] if w == 0 else v[lo] * (1 - w) + v[hi] * w)
    return out


def quantile_aggregate(ssts, schema: pa.Schema, num_pk: int, preds=(), group_col: int = 0, ts_col: int = -1, window_ms: int = 0,
                       value_col: int = 2, mode: int = 0, quantiles=(0.5,)) -> pa.Table:
    """The table `Engine.scan_quantile_aggregate` returns for the same arguments (`schema`: the full storage schema)."""
    res = oracle.scan(ssts, schema, num_pk, preds)
    has_ts = ts_col >= 0 and window_ms > 0
    vt = schema.field(value_col).type
    groups = []                       # [key, bucket, count, values]
    index = {}
    for b in res.batches:
        n = b.num_rows
        g = b.column(group_col).to_pylist() if group_col >= 0 else [None] * n
        t = b.column(ts_col).to_pylist() if has_ts else [0] * n
        v = b.column(value_col).to_pylist()
        for key, ts, val in zip(g, t, v):
            if has_ts and ts >= 1 << 63:
                ts -= 1 << 64                      # the time column widened to i64
            bucket = _trunc_div(ts, window_ms) * window_ms if has_ts else 0
            if mode == HG_AGG_HASH:
                grp = index.get((key, bucket))
                if grp is None:
                    grp = index[(key, bucket)] = [key, bucket, 0, []]
                    groups.append(grp)
            else:
                if not groups or (groups[-1][0], groups[-1][1]) != (key, bucket):
                    groups.append([key, bucket, 0, []])
                grp = groups[-1]
            grp[2] += 1
            if val is not None:
                grp[3].append(val)
    if mode == HG_AGG_HASH:
        kt = schema.field(group_col).type if group_col >= 0 else pa.uint64()
        groups.sort(key=lambda gr: (order_key(gr[0], kt) if gr[0] is not None else 0, gr[1]))
    cols, names = [], []
    if group_col >= 0:
        cols.append(pa.array([gr[0] for gr in groups], schema.field(group_col).type))
        names.append(schema.field(group_col).name)
    if has_ts:
        cols.append(pa.array([gr[1] for gr in groups], pa.int64()))
        names.append("bucket")
    cols.append(pa.array([gr[2] for gr in groups], pa.uint64()))
    names.append("count")
    per_group = [quantiles_of(gr[3], vt, quantiles) for gr in groups]
    for j in range(len(quantiles)):
        cols.append(pa.array([r[j] for r in per_group], pa.float64()))
        names.append("quantile_%d" % j)
    return pa.Table.from_arrays(cols, names=names)
