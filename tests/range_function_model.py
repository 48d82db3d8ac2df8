"""TEST INFRASTRUCTURE: the model of `hg_scan_range_function` / `hg_scan_range_function_by_map`.  A literal Python transcription of the
definitions in include/horae_gpu.h over the windows of range_model.py (the C oracle's deduplicated stream); it uses nothing of the library.

Python floats are IEEE doubles and Python never fuses a multiply with an add, so every operation below is rounded on its own, as the
definitions require: the model is exact, bit for bit."""
from __future__ import annotations

import pyarrow as pa

from range_model import _windows

(RATE, INCREASE, DELTA, IRATE, IDELTA, RESETS, CHANGES, COUNT_OVER_TIME, SUM_OVER_TIME, MIN_OVER_TIME, MAX_OVER_TIME,
 LAST_OVER_TIME) = range(12)
ALL_FNS = tuple(range(12))
NAMES = ("rate", "increase", "delta", "irate", "idelta", "resets", "changes", "count_over_time", "sum_over_time", "min_over_time",
         "max_over_time", "last_over_time")


def seconds(range_ms: int) -> float:
    """Go's Duration.Seconds of range_ms milliseconds: whole seconds plus the nanoseconds / 1e9"""
    return float(range_ms // 1000) + float((range_ms % 1000) * 1000000) / 1e9


def extrapolation(t: int, range_ms: int, samples, counter: bool):
    """the intermediates of Prometheus 3's extrapolatedRate (m >= 2, T_(m-1) != T_0): result, sampled, dStart (after the threshold and
    the zero-point clamp) and dEnd (after the threshold)"""
    (t0, v0), (tl, vl) = samples[0], samples[-1]
    result = vl - v0
    if counter:
        prev = v0
        for _, x in samples[1:]:
            if x < prev:
                result = result + prev
            prev = x
    d_start = float(t0 - (t - range_ms)) / 1000
    d_end = float(t - tl) / 1000
    sampled = float(tl - t0) / 1000
    avg = sampled / float(len(samples) - 1)
    thr = avg * 1.1
    if d_start >= thr:
        d_start = avg / 2
    d_zero = None
    if counter and result > 0 and v0 >= 0:
        d_zero = sampled * (v0 / result)
        if d_zero < d_start:
            d_start = d_zero
    if d_end >= thr:
        d_end = avg / 2
    return result, sampled, d_start, d_end, d_zero


def fn_value(fn: int, t: int, range_ms: int, ts, vals):
    """the value of range function fn over one window's rows (ts, vals in stream order; None = a NULL value), or None: no value"""
    s = [(T, float(V)) for T, V in zip(ts, vals) if V is not None]
    m = len(s)
    if m == 0:
        return None
    if fn in (RATE, INCREASE, DELTA):
        if m < 2 or s[-1][0] == s[0][0]:
            return None
        result, sampled, d_start, d_end, _ = extrapolation(t, range_ms, s, fn != DELTA)
        ext = sampled + d_start
        ext = ext + d_end
        factor = ext / sampled
        if fn == RATE:
            factor = factor / seconds(range_ms)
        return result * factor
    if fn in (IRATE, IDELTA):
        if m < 2:
            return None
        (ta, va), (tb, vb) = s[-2], s[-1]
        if tb == ta:
            return None
        if fn == IDELTA:
            return vb - va
        return (vb if vb < va else vb - va) / (float(tb - ta) / 1000)
    vs = [v for _, v in s]
    if fn == RESETS:
        return float(sum(1 for i in range(1, m) if vs[i] < vs[i - 1]))
    if fn == CHANGES:
        return float(sum(1 for i in range(1, m) if not (vs[i] == vs[i - 1] or (vs[i] != vs[i] and vs[i - 1] != vs[i - 1]))))
    if fn == COUNT_OVER_TIME:
        return float(m)
    if fn == LAST_OVER_TIME:
        return vs[-1]
    total, mn, mx = 0.0, None, None
    for x in vs:
        total += x
        if mn is None or x < mn:
            mn = x
        if mx is None or x > mx:
            mx = x
    return {SUM_OVER_TIME: total, MIN_OVER_TIME: mn, MAX_OVER_TIME: mx}[fn]


def function_windows(ssts, schema: pa.Schema, num_pk: int, fn: int, preds=(), start_ms=0, end_ms=0, step_ms=1, range_ms=1, value_col=2):
    """[(series key, t, value)] of the windows with a value, in (series, t) order"""
    out = []
    for key, t, ts, vals in _windows(ssts, schema, num_pk, preds, start_ms, end_ms, step_ms, range_ms, value_col):
        v = fn_value(fn, t, range_ms, ts, vals)
        if v is not None:
            out.append((key, t, v))
    return out


def range_function(ssts, schema: pa.Schema, num_pk: int, fn: int, preds=(), start_ms=0, end_ms=0, step_ms=1, range_ms=1, value_col=2) -> pa.Table:
    """The table `Engine.scan_range_function` returns for the same arguments (`schema`: the full storage schema)."""
    rows = function_windows(ssts, schema, num_pk, fn, preds, start_ms, end_ms, step_ms, range_ms, value_col)
    return pa.Table.from_arrays([pa.array([r[0] for r in rows], schema.field(0).type), pa.array([r[1] for r in rows], pa.int64()),
                                 pa.array([r[2] for r in rows], pa.float64())], names=[schema.field(0).name, "t", "value"])


def group_rows(rows, keys, groups):
    """per (group, t) of the windows `rows` ((series, t, value) in series order) whose series is in the map: count, the sequential sum in
    series order, min / max with hg_scan_aggregate's rule (the first value starts both); sorted by (group, t)"""
    gmap = {}
    for k, g in zip(keys, groups):
        gmap[int(k)] = int(g)
    acc = {}
    for key, t, v in rows:
        if key not in gmap:
            continue
        a = acc.setdefault((gmap[key], t), [0, 0.0, None, None])
        a[0] += 1
        a[1] += v
        if a[2] is None or v < a[2]:
            a[2] = v
        if a[3] is None or v > a[3]:
            a[3] = v
    return [(g, t, *acc[(g, t)]) for g, t in sorted(acc)]


def range_function_by_map(ssts, schema: pa.Schema, num_pk: int, fn: int, keys, groups, preds=(), start_ms=0, end_ms=0, step_ms=1, range_ms=1,
                          value_col=2) -> pa.Table:
    """The table `Engine.scan_range_function_by_map` returns for the same arguments: the per-series values of `range_function` (the rows
    of series outside the map filtered first), summed by group."""
    rows = function_windows(ssts, schema, num_pk, fn, preds, start_ms, end_ms, step_ms, range_ms, value_col)
    out = group_rows(rows, keys, groups)
    names = ["group", "t", "count", "sum", "min", "max"]
    types = [pa.uint32(), pa.int64(), pa.uint64(), pa.float64(), pa.float64(), pa.float64()]
    return pa.Table.from_arrays([pa.array([r[i] for r in out], types[i]) for i in range(6)], names=names)
