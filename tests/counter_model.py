"""TEST INFRASTRUCTURE: the model of `hg_scan_counter_aggregate`.  A plain sequential Python restatement of the counter partials per
(series, bucket) over the deduplicated stream of the C oracle (`oracle.scan`); it uses nothing of the library.

Per group, over its non-NULL values v1..vm in stream order, each as an f64 (Python's float(int) rounds to nearest, as the C conversion
does):  resets = #{i >= 2 : v_i < v_(i-1)},  increase = 0.0 then += (v_i < v_(i-1) ? v_i : v_i - v_(i-1)), in order."""
from __future__ import annotations

import pyarrow as pa

from oracle import oracle


def _trunc_div(a: int, b: int) -> int:
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def counter_aggregate(ssts, schema: pa.Schema, num_pk: int, preds=(), group_col: int = 0, ts_col: int = 1, window_ms: int = 0,
                      value_col: int = 2) -> pa.Table:
    """The table `Engine.scan_counter_aggregate` returns for the same arguments (`schema`: the full storage schema)."""
    res = oracle.scan(ssts, schema, num_pk, preds)
    keys, buckets, counts, first_ts, first_v, last_ts, last_v, incs, resets = ([] for _ in range(9))
    cur = None
    for b in res.batches:
        g = b.column(group_col).to_pylist()
        t = b.column(ts_col).to_pylist()
        v = b.column(value_col).to_pylist()
        for key, ts, val in zip(g, t, v):
            if ts >= 1 << 63:
                ts -= 1 << 64                      # the time column widened to i64
            bucket = _trunc_div(ts, window_ms) * window_ms if window_ms > 0 else 0
            if cur != (key, bucket):
                cur = (key, bucket)
                keys.append(key)
                buckets.append(bucket)
                counts.append(0)
                first_ts.append(None)
                first_v.append(None)
                last_ts.append(None)
                last_v.append(None)
                incs.append(0.0)
                resets.append(0)
            counts[-1] += 1
            if val is None:
                continue
            x = float(val)
            if first_v[-1] is None:
                first_ts[-1], first_v[-1] = ts, x
            else:
                prev = last_v[-1]
                if x < prev:
                    incs[-1] += x
                    resets[-1] += 1
                else:
                    incs[-1] += x - prev
            last_ts[-1], last_v[-1] = ts, x
    cols = [pa.array(keys, schema.field(group_col).type)]
    names = [schema.field(group_col).name]
    if window_ms > 0:
        cols.append(pa.array(buckets, pa.int64()))
        names.append("bucket")
    cols += [pa.array(counts, pa.uint64()), pa.array(first_ts, pa.int64()), pa.array(first_v, pa.float64()), pa.array(last_ts, pa.int64()),
             pa.array(last_v, pa.float64()), pa.array(incs, pa.float64()), pa.array(resets, pa.uint64())]
    names += ["count", "first_ts", "first_value", "last_ts", "last_value", "increase", "resets"]
    return pa.Table.from_arrays(cols, names=names)
