"""SST writer with the reference's writer properties + deterministic synthetic metric data.

`write_sst` restates `ObjectBasedStorage::write_batch` + `build_write_props` (storage.rs:189-225, 258-298):
rows sorted by primary key, `__seq__`/`__reserved__` appended (types.rs:219-239), Parquet with row groups of
`max_row_group_size`, dictionary off, PLAIN, Snappy by default (config.rs:120-133), `sorting_columns` = PKs.
The write path is not on the accelerated hot path (SURVEY §8f rank 1/3); it uses pyarrow's Parquet writer, an
independent implementation of the same format parquet-rs 53.2 writes.

`synth_*` is the measurement data of SURVEY §8(d): splitmix64 streams, seed 42.
"""
from __future__ import annotations

import io
from typing import List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from .config import ParquetCompression, WriteConfig, resolve_bloom_filters
from .types import StorageSchema

T0_MS = 1_700_000_000_000
SEED = 42
_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(x: np.ndarray) -> np.ndarray:
    """Vectorised splitmix64 finaliser over uint64 (wrapping arithmetic)."""
    with np.errstate(over="ignore"):
        z = (x + np.uint64(0x9E3779B97F4A7C15)).astype(np.uint64)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def synth_columns(series_lo: int, series_hi: int, points: int, delta_ms: int, seed: int = SEED,
                  point_lo: int = 0):
    """Rows for series in [series_lo, series_hi) × points j in [point_lo, point_lo+points), sorted by (series_id, ts).

    ts = T0 + j·Δ + jitter, jitter ∈ [0, Δ/2) ; value ∈ [0,1) ; tag = s mod 16   (SURVEY §8d).
    """
    s = np.arange(series_lo, series_hi, dtype=np.uint64)
    j = np.arange(point_lo, point_lo + points, dtype=np.uint64)
    sid = np.repeat(s, points)
    jj = np.tile(j, len(s))
    with np.errstate(over="ignore"):
        h1 = splitmix64(np.uint64(seed) ^ (sid << np.uint64(32)) ^ jj)
    half = max(delta_ms // 2, 1)
    jitter = (h1 % np.uint64(half)).astype(np.int64)
    ts = np.int64(T0_MS) + jj.astype(np.int64) * np.int64(delta_ms) + jitter
    h2 = splitmix64(h1)
    value = (h2 >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53))
    tag = (sid % np.uint64(16)).astype(np.uint32)
    return sid, ts, value, tag


METRIC_SCHEMA = pa.schema(
    [
        pa.field("series_id", pa.uint64(), True),
        pa.field("ts", pa.int64(), True),
        pa.field("value", pa.float64(), True),
        pa.field("tag", pa.uint32(), True),
    ]
)


def metric_storage_schema() -> StorageSchema:
    """Canonical metric-data schema of SURVEY §8: pk = (series_id, ts); values = (value, tag)."""
    return StorageSchema.try_new(METRIC_SCHEMA, 2)


def _writer_kwargs(schema: StorageSchema, cfg: WriteConfig) -> dict:
    """`build_write_props` (storage.rs:258-298) expressed as pyarrow writer arguments."""
    kw = dict(
        row_group_size=cfg.max_row_group_size,
        write_batch_size=cfg.write_bacth_size,
        use_dictionary=cfg.enable_dict,
        compression=cfg.compression,
        write_statistics=True,
        data_page_version="1.0",
        store_schema=True,
    )
    if cfg.enable_sorting_columns:
        kw["sorting_columns"] = [pq.SortingColumn(i, False, True) for i in range(schema.num_primary_keys)]
    col_enc = {}
    col_comp = {}
    col_dict = []
    names = schema.arrow_schema.names
    if cfg.encoding != "PLAIN":
        col_enc = {n: cfg.encoding for n in names}
    if cfg.column_options:
        for name, opt in cfg.column_options.items():
            if opt.encoding is not None:
                col_enc[name] = opt.encoding
            if opt.compression is not None:
                col_comp[name] = opt.compression
            if opt.enable_dict:
                col_dict.append(name)
    if col_enc:
        kw["column_encoding"] = col_enc
        kw["use_dictionary"] = col_dict if col_dict else False
    elif col_dict:
        kw["use_dictionary"] = col_dict
    if col_comp:
        comp = {n: cfg.compression for n in names}
        comp.update(col_comp)
        kw["compression"] = comp
    blooms = resolve_bloom_filters(cfg, schema.arrow_schema)
    if blooms is not None:
        # parquet-rs's BloomFilterProperties::default (ndv 1,000,000, fpp 0.05): a 1 MiB bitset per column chunk
        kw["bloom_filter_options"] = {n: {"ndv": 1_000_000, "fpp": 0.05} for n, b in zip(names, blooms) if b}
    return kw


def sort_batch(schema: StorageSchema, batch: pa.RecordBatch) -> pa.RecordBatch:
    """`sort_batch` (storage.rs:244-256): sort by PK columns ascending, nulls first."""
    keys = [(schema.arrow_schema.names[i], "ascending") for i in range(schema.num_primary_keys)]
    tbl = pa.Table.from_batches([batch])
    idx = pa.compute.sort_indices(tbl, sort_keys=keys, null_placement="at_start")
    return tbl.take(idx).combine_chunks().to_batches()[0] if batch.num_rows else batch


def write_sst(schema: StorageSchema, batch: pa.RecordBatch, seq: int, cfg: Optional[WriteConfig] = None,
              presorted: bool = False) -> bytes:
    """One SST's bytes for a user-schema batch (storage.rs:189-225). `seq` is the file id (storage.rs:207-208)."""
    cfg = cfg or WriteConfig()
    if not presorted:
        batch = sort_batch(schema, batch)
    full = schema.fill_builtin_columns(batch, seq)
    if full.num_rows == 0:
        full = pa.RecordBatch.from_arrays(
            [pa.array([], f.type) for f in schema.arrow_schema], schema=schema.arrow_schema)
    sink = io.BytesIO()
    pq.write_table(pa.Table.from_batches([full]), sink, **_writer_kwargs(schema, cfg))
    return sink.getvalue()


def write_sst_with_seq(schema: StorageSchema, batch_with_builtin: pa.RecordBatch,
                       cfg: Optional[WriteConfig] = None) -> bytes:
    """SST from a batch that already carries `__seq__`/`__reserved__` (what compaction writes, executor.rs:173-191)."""
    cfg = cfg or WriteConfig()
    sink = io.BytesIO()
    pq.write_table(pa.Table.from_batches([batch_with_builtin]), sink, **_writer_kwargs(schema, cfg))
    return sink.getvalue()


def synth_sst(series_lo: int, series_hi: int, points: int, delta_ms: int, seq: int,
              compression: str = ParquetCompression.Snappy, seed: int = SEED, with_tag: bool = True,
              row_group: int = 8192) -> Tuple[bytes, int]:
    """One synthetic metric SST covering a contiguous series range. Returns (bytes, num_rows)."""
    sid, ts, value, tag = synth_columns(series_lo, series_hi, points, delta_ms, seed)
    schema = metric_storage_schema()
    batch = pa.RecordBatch.from_arrays(
        [pa.array(sid), pa.array(ts), pa.array(value), pa.array(tag)], schema=METRIC_SCHEMA)
    cfg = WriteConfig(compression=compression, max_row_group_size=row_group)
    return write_sst(schema, batch, seq, cfg, presorted=True), len(sid)


def synth_overlapping_ssts(n_files: int, series: int, points: int, delta_ms: int, keep_frac: float,
                           compression: str = ParquetCompression.Snappy, seed: int = SEED,
                           base_seq: int = 1000) -> List[Tuple[bytes, int, int]]:
    """Config-5 style inputs (SURVEY §8d): every file samples the same series×points PK universe
    (each PK kept with probability `keep_frac`, per-file hash), values differ per file, `__seq__` = file id.
    Returns [(bytes, num_rows, seq)]."""
    schema = metric_storage_schema()
    out = []
    sid, ts, value, tag = synth_columns(0, series, points, delta_ms, seed)
    thresh = np.uint64(int(keep_frac * float(1 << 64)) - 1 if keep_frac < 1.0 else 0xFFFFFFFFFFFFFFFF)
    for f in range(n_files):
        seq = base_seq + f
        with np.errstate(over="ignore"):
            h = splitmix64((sid << np.uint64(20)) ^ ts.astype(np.uint64) ^ (np.uint64(seq) * np.uint64(0x9E3779B97F4A7C15)))
        keep = h <= thresh
        v = (splitmix64(h) >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53))
        batch = pa.RecordBatch.from_arrays(
            [pa.array(sid[keep]), pa.array(ts[keep]), pa.array(v[keep]), pa.array(tag[keep])], schema=METRIC_SCHEMA)
        data = write_sst(schema, batch, seq, WriteConfig(compression=compression), presorted=True)
        out.append((data, int(keep.sum()), seq))
    return out
