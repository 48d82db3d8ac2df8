"""Mirror of `columnar_storage::config` (config.rs:26-172) — only what defines the SST format (S1)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple


class ParquetEncoding:  # config.rs:54-75
    Plain = "PLAIN"
    Rle = "RLE"
    DeltaBinaryPacked = "DELTA_BINARY_PACKED"
    DeltaLengthByteArray = "DELTA_LENGTH_BYTE_ARRAY"
    DeltaByteArray = "DELTA_BYTE_ARRAY"
    RleDictionary = "RLE_DICTIONARY"


class ParquetCompression:  # config.rs:79-94
    Uncompressed = "none"
    Snappy = "snappy"
    Zstd = "zstd"


@dataclass
class ColumnOptions:  # config.rs:98-103
    enable_dict: Optional[bool] = None
    enable_bloom_filter: Optional[bool] = None
    encoding: Optional[str] = None
    compression: Optional[str] = None


@dataclass
class WriteConfig:  # config.rs:107-133 (defaults 120-133)
    max_row_group_size: int = 8192
    write_bacth_size: int = 1024  # sic — the reference's spelling
    enable_sorting_columns: bool = True
    enable_dict: bool = False
    enable_bloom_filter: bool = False
    encoding: str = ParquetEncoding.Plain
    compression: str = ParquetCompression.Snappy
    column_options: Optional[Dict[str, ColumnOptions]] = None


_GPU_CODECS = ("none", "uncompressed", "snappy", "zstd")


def resolve_column_options(cfg: WriteConfig, arrow_schema) -> Optional[List[Tuple[str, bool, str]]]:
    """The writer options of every column of the storage schema (builtin columns included), as `build_write_props` (storage.rs:258-298)
    resolves them: `column_options[name]` overrides the table-wide field.  One (encoding, dictionary, codec) per column, the form
    `Engine.compact_to_sst(columns=...)` / `Engine.write_batch(columns=...)` take — or None when some column needs what the GPU writer does
    not implement: a Binary column, an encoding other than PLAIN / DELTA_BINARY_PACKED (RLE_DICTIONARY is not a fallback encoding;
    a dictionary is `enable_dict`), DELTA on a float column, or a codec other than Uncompressed / Snappy / Zstd."""
    import pyarrow as pa
    out = []
    opts = cfg.column_options or {}
    for f in arrow_schema:
        o = opts.get(f.name) or ColumnOptions()
        enc = o.encoding if o.encoding is not None else cfg.encoding
        dictionary = o.enable_dict if o.enable_dict is not None else cfg.enable_dict
        codec = str(o.compression if o.compression is not None else cfg.compression).lower()
        if pa.types.is_binary(f.type) or codec not in _GPU_CODECS:
            return None
        if enc == ParquetEncoding.DeltaBinaryPacked:
            if not pa.types.is_integer(f.type):
                return None
        elif enc != ParquetEncoding.Plain:
            return None
        out.append((enc, bool(dictionary), codec))
    return out


def resolve_bloom_filters(cfg: WriteConfig, arrow_schema) -> Optional[List[bool]]:
    """Which columns of the storage schema (builtin columns included) get a bloom filter, as `build_write_props` (storage.rs:272, 285-288)
    resolves it: `column_options[name].enable_bloom_filter` overrides the table-wide `enable_bloom_filter`.  One flag per column, the form
    `Engine.compact_to_sst(bloom_filters=...)` / `Engine.write_batch(bloom_filters=...)` take — or None when no column wants one."""
    opts = cfg.column_options or {}
    out = []
    for f in arrow_schema:
        o = opts.get(f.name) or ColumnOptions()
        out.append(bool(o.enable_bloom_filter if o.enable_bloom_filter is not None else cfg.enable_bloom_filter))
    return out if any(out) else None


@dataclass
class SchedulerConfig:  # config.rs:26-50 (caller of the compaction path; kept for its limits)
    memory_limit: int = 2 << 30
    new_sst_max_size: int = 1 << 30
    input_sst_max_num: int = 30
    input_sst_min_num: int = 5


@dataclass
class StorageConfig:  # config.rs:157-164
    write: WriteConfig = field(default_factory=WriteConfig)
    scheduler: SchedulerConfig = field(default_factory=SchedulerConfig)
    update_mode: int = 0
