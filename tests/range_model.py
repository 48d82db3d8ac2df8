"""TEST INFRASTRUCTURE: the model of `hg_scan_range_aggregate` / `hg_scan_range_quantile_aggregate`.  A plain Python restatement of PromQL
range windows over the deduplicated stream of the C oracle (`oracle.scan`); it uses nothing of the library.

Evaluation times t_j = start + j * step, j = 0 .. (end - start) // step (one step when start == end).  Per series (a run of equal keys in
the stream), per t_j, the window is the series' rows with t_j - range < ts <= t_j; a window without rows does not appear.  Over a window's
rows in stream order: count (NULL values included); sum / min / max of the non-NULL values as f64 (0 / +inf / -inf without one); the
counter partials of counter_model.py (first / last non-NULL sample, increase, resets); or the quantiles of quantile_model.py."""
from __future__ import annotations

import bisect

import pyarrow as pa

from oracle import oracle
from quantile_model import quantiles_of

INF = float("inf")


def steps(start_ms: int, end_ms: int, step_ms: int) -> int:
    return 1 if start_ms == end_ms else (end_ms - start_ms) // step_ms + 1


def _series(res, value_col: int):
    """[(key, [ts...], [value...])] in stream order"""
    out = []
    for b in res.batches:
        for key, ts, val in zip(b.column(0).to_pylist(), b.column(1).to_pylist(), b.column(value_col).to_pylist()):
            if not out or out[-1][0] != key:
                out.append((key, [], []))
            out[-1][1].append(ts)
            out[-1][2].append(val)
    return out


def _window_steps(ts, start_ms, step_ms, range_ms, n):
    """the steps j whose window holds one of the times ts (sorted), in order"""
    js = []
    last = -1
    for x in ts:
        lo = max(0, -((start_ms - x) // step_ms))                  # ceil((x - start) / step)
        hi = min(n - 1, (x + range_ms - 1 - start_ms) // step_ms)   # floor
        for j in range(max(lo, last + 1), hi + 1):
            js.append(j)
        last = max(last, hi)
    return js


def _windows(ssts, schema, num_pk, preds, start_ms, end_ms, step_ms, range_ms, value_col):
    res = oracle.scan(ssts, schema, num_pk, preds)
    if start_ms == end_ms:
        step_ms = 1
    n = steps(start_ms, end_ms, step_ms)
    for key, ts, vals in _series(res, value_col):
        for j in _window_steps(ts, start_ms, step_ms, range_ms, n):
            t = start_ms + j * step_ms
            a, b = bisect.bisect_right(ts, t - range_ms), bisect.bisect_right(ts, t)
            if a < b:
                yield key, t, ts[a:b], vals[a:b]


def range_aggregate(ssts, schema: pa.Schema, num_pk: int, preds=(), start_ms=0, end_ms=0, step_ms=1, range_ms=1, value_col=2) -> pa.Table:
    """The table `Engine.scan_range_aggregate` returns for the same arguments (`schema`: the full storage schema)."""
    cols = {n: [] for n in ("key", "t", "count", "sum", "min", "max", "first_ts", "first_value", "last_ts", "last_value", "increase", "resets")}
    for key, t, ts, vals in _windows(ssts, schema, num_pk, preds, start_ms, end_ms, step_ms, range_ms, value_col):
        s, mn, mx = 0.0, INF, -INF
        first_ts = first_v = last_ts = last_v = None
        inc, resets = 0.0, 0
        for x_ts, val in zip(ts, vals):
            if val is None:
                continue
            x = float(val)
            s += x
            if first_v is None or x < mn:
                mn = x
            if first_v is None or x > mx:
                mx = x
            if first_v is None:
                first_ts, first_v = x_ts, x
            elif x < last_v:
                inc += x
                resets += 1
            else:
                inc += x - last_v
            last_ts, last_v = x_ts, x
        for name, v in (("key", key), ("t", t), ("count", len(ts)), ("sum", s), ("min", mn), ("max", mx), ("first_ts", first_ts),
                        ("first_value", first_v), ("last_ts", last_ts), ("last_value", last_v), ("increase", inc), ("resets", resets)):
            cols[name].append(v)
    types = {"t": pa.int64(), "count": pa.uint64(), "first_ts": pa.int64(), "last_ts": pa.int64(), "resets": pa.uint64()}
    arrays = [pa.array(cols["key"], schema.field(0).type)]
    names = [schema.field(0).name]
    for name in list(cols)[1:]:
        arrays.append(pa.array(cols[name], types.get(name, pa.float64())))
        names.append(name)
    return pa.Table.from_arrays(arrays, names=names)


def range_quantile_aggregate(ssts, schema: pa.Schema, num_pk: int, preds=(), start_ms=0, end_ms=0, step_ms=1, range_ms=1, value_col=2,
                             quantiles=(0.5,)) -> pa.Table:
    """The table `Engine.scan_range_quantile_aggregate` returns for the same arguments."""
    vt = schema.field(value_col).type
    keys, times, counts, per = [], [], [], []
    for key, t, ts, vals in _windows(ssts, schema, num_pk, preds, start_ms, end_ms, step_ms, range_ms, value_col):
        keys.append(key)
        times.append(t)
        counts.append(len(ts))
        per.append(quantiles_of([v for v in vals if v is not None], vt, quantiles))
    arrays = [pa.array(keys, schema.field(0).type), pa.array(times, pa.int64()), pa.array(counts, pa.uint64())]
    names = [schema.field(0).name, "t", "count"]
    for j in range(len(quantiles)):
        arrays.append(pa.array([r[j] for r in per], pa.float64()))
        names.append("quantile_%d" % j)
    return pa.Table.from_arrays(arrays, names=names)
