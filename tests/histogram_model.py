"""TEST INFRASTRUCTURE: the model of `hg_scan_histogram_quantile`.  A literal Python transcription of the definition in include/horae_gpu.h
over the per-series values of range_function_model.py (the C oracle's deduplicated stream); it uses nothing of the library.

Python floats are IEEE doubles and Python never fuses a multiply with an add, so every operation below is rounded on its own: the model is
exact, bit for bit.  `STEPS` counts which step of the definition decided each value, so that tests can assert that a case reaches the
branch it is written for."""
from __future__ import annotations

from collections import Counter

import numpy as np
import pyarrow as pa

from range_function_model import function_windows

MIN_NORMAL = 2.0 ** -1022
MAX_F64 = 1.7976931348623157e308
NAN = float("nan")
INF = float("inf")

# which step decided a value (or, for "fixup_*", happened): reset by the caller between cases
STEPS = Counter()


def _div(a: float, b: float) -> float:
    """IEEE division (Python raises on a zero divisor)"""
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def almost_equal(a: float, b: float) -> bool:
    """util/almost.Equal(a, b, 1e-12)"""
    if (a != a and b != b) or a == b:
        return True
    s = abs(a) + abs(b)
    d = abs(a - b)
    if a == 0 or b == 0 or s < MIN_NORMAL:
        return d < 1e-12 * MIN_NORMAL
    m = s if (s != s or s < MAX_F64) else MAX_F64          # Go's math.Min keeps a NaN
    return d / m < 1e-12


def fix_up(counts):
    """step 3 in place; returns forced_monotonic"""
    forced = False
    prev = counts[0]
    for i in range(1, len(counts)):
        cur = counts[i]
        if cur == prev:
            continue
        if almost_equal(prev, cur):
            counts[i] = prev
            STEPS["fixup_small_delta"] += 1
            continue
        if cur < prev:
            counts[i] = prev
            forced = True
            STEPS["fixup_forced"] += 1
            continue
        prev = cur
    return forced


def bucket_quantiles(buckets, qs):
    """buckets: [(upper bound, count)] with distinct bounds in ascending order; returns (forced_monotonic, [value per q])"""
    n = len(buckets)
    u = [b for b, _ in buckets]
    c = [x for _, x in buckets]
    if not (u[-1] == INF):
        STEPS["no_inf"] += len(qs)
        return 0, [NAN] * len(qs)
    forced = fix_up(c)
    if n < 2:
        STEPS["inf_alone"] += len(qs)
        return int(forced), [NAN] * len(qs)
    obs = c[n - 1]
    if obs == 0:
        STEPS["obs_zero"] += len(qs)
        return int(forced), [NAN] * len(qs)
    out = []
    for q in qs:
        rank = q * obs
        lo, hi = 0, n - 1
        while lo < hi:
            h = (lo + hi) // 2
            if not (c[h] >= rank):
                lo = h + 1
            else:
                hi = h
        b = lo
        if b == n - 1:
            STEPS["b_last"] += 1
            out.append(u[n - 2])
            continue
        if b == 0 and u[0] <= 0:
            STEPS["b0_nonpositive"] += 1
            out.append(u[0])
            continue
        start, end, cnt = 0.0, u[b], c[b]
        if b > 0:
            start = u[b - 1]
            cnt = cnt - c[b - 1]
            rank = rank - c[b - 1]
            STEPS["interp_later"] += 1
        else:
            STEPS["interp_first"] += 1
        out.append(start + (end - start) * _div(rank, cnt))
    return int(forced), out


def bucket_sums(rows, keys, groups, bounds):
    """{(group, t): {bound: the sequential sum in series order}} of the windows `rows` ((series, t, value) in series order) whose series is in
    the map; -0.0 and +0.0 are one bound (+0.0)"""
    pair = {}
    for k, g, b in zip(keys, groups, bounds):
        pair[int(k)] = (int(g), float(b) + 0.0)
    acc = {}
    for key, t, v in rows:
        if key not in pair:
            continue
        g, b = pair[key]
        cell = acc.setdefault((g, t), {})
        cell[b] = cell.get(b, 0.0) + v
    return acc


def histogram_rows(rows, keys, groups, bounds, qs):
    """[(group, t, forced_monotonic, [quantiles])] sorted by (group, t)"""
    acc = bucket_sums(rows, keys, groups, bounds)
    out = []
    for g, t in sorted(acc):
        cell = acc[(g, t)]
        forced, vals = bucket_quantiles(sorted(cell.items()), qs)
        out.append((g, t, forced, vals))
    return out


def histogram_table(out, nq) -> pa.Table:
    arrays = [pa.array([r[0] for r in out], pa.uint32()), pa.array([r[1] for r in out], pa.int64()), pa.array([r[2] for r in out], pa.uint8())]
    names = ["group", "t", "forced_monotonic"]
    for j in range(nq):
        arrays.append(pa.array([r[3][j] for r in out], pa.float64()))
        names.append("quantile_%d" % j)
    return pa.Table.from_arrays(arrays, names=names)


def histogram_quantile(ssts, schema: pa.Schema, num_pk: int, fn: int, keys, groups, bounds, qs, preds=(), start_ms=0, end_ms=0, step_ms=1,
                       range_ms=1, value_col=2) -> pa.Table:
    """The table `Engine.scan_histogram_quantile` returns for the same arguments (`schema`: the full storage schema)."""
    rows = function_windows(ssts, schema, num_pk, fn, preds, start_ms, end_ms, step_ms, range_ms, value_col)
    return histogram_table(histogram_rows(rows, keys, groups, bounds, qs), len(qs))
