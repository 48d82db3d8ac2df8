"""TEST INFRASTRUCTURE: the model of `hg_scan_range_function_topk`.  A literal Python transcription of the definition in
include/horae_gpu.h over range_function_model.py's per-series values (the C oracle's deduplicated stream); it uses nothing of the library.

Per (group, t): the series mapped to the group that have a value at t, in series-key (stream) order, sorted by Python's stable sort with
the key (isnan(v), -v) for HG_TOPK or (isnan(v), v) for HG_BOTTOMK (NaN last in both; values equal under IEEE, -0.0 and +0.0 or two
NaNs, keep series order), then the first k."""
from __future__ import annotations

import math

import pyarrow as pa

from range_function_model import function_windows

TOPK, BOTTOMK = 0, 1


def rank_key(v: float, order: int):
    if math.isnan(v):
        return (True, 0.0)
    return (False, -v if order == TOPK else v)


def topk_rows(rows, keys, groups, k: int, order: int):
    """[(group, t, series key, value)] of the windows `rows` ((series, t, value) in series order) whose series is in the map, the first k
    per (group, t) in rank order, sorted by (group, t, rank)"""
    gmap = {int(key): int(g) for key, g in zip(keys, groups)}
    seg = {}
    for key, t, v in rows:
        if key in gmap:
            seg.setdefault((gmap[key], t), []).append((key, v))
    out = []
    for g, t in sorted(seg):
        for key, v in sorted(seg[(g, t)], key=lambda e: rank_key(e[1], order))[:k]:
            out.append((g, t, key, v))
    return out


def range_function_topk(ssts, schema: pa.Schema, num_pk: int, fn: int, k: int, keys, groups, order=TOPK, preds=(), start_ms=0, end_ms=0,
                        step_ms=1, range_ms=1, value_col=2) -> pa.Table:
    """The table `Engine.scan_range_function_topk` returns for the same arguments (`schema`: the full storage schema)."""
    rows = function_windows(ssts, schema, num_pk, fn, preds, start_ms, end_ms, step_ms, range_ms, value_col)
    out = topk_rows(rows, keys, groups, k, order)
    return pa.Table.from_arrays([pa.array([r[0] for r in out], pa.uint32()), pa.array([r[1] for r in out], pa.int64()),
                                 pa.array([r[2] for r in out], schema.field(0).type), pa.array([r[3] for r in out], pa.float64())],
                                names=["group", "t", schema.field(0).name, "value"])
