"""ctypes binding of libhorae_gpu.so (include/horae_gpu.h).  Fails loudly when the CUDA library is missing:
there is no CPU fallback anywhere in this package."""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libhorae_gpu.so")

HG_TYPES = {pa.uint8(): 0, pa.int8(): 1, pa.uint16(): 2, pa.int16(): 3, pa.uint32(): 4, pa.int32(): 5,
            pa.uint64(): 6, pa.int64(): 7, pa.float32(): 8, pa.float64(): 9, pa.binary(): 10}
HG_OPS = {"eq": 0, "ne": 1, "lt": 2, "le": 3, "gt": 4, "ge": 5, "in": 6, "in_set": 7}
HG_MAX_IN_SET = 1 << 24
HG_FLAG_NO_PRUNING = 1
HG_FLAG_NO_FUSED = 2
HG_FLAG_NO_LATE_MATERIALIZATION = 4
HG_FLAG_PAIRWISE_MERGE = 8
HG_FLAG_NO_BLOOM_FILTER = 16
HG_AGG_RUNS, HG_AGG_HASH = 0, 1
# hg_range_fn: the PromQL range functions of scan_range_function / scan_range_function_by_map
(HG_FN_RATE, HG_FN_INCREASE, HG_FN_DELTA, HG_FN_IRATE, HG_FN_IDELTA, HG_FN_RESETS, HG_FN_CHANGES, HG_FN_COUNT_OVER_TIME, HG_FN_SUM_OVER_TIME,
 HG_FN_MIN_OVER_TIME, HG_FN_MAX_OVER_TIME, HG_FN_LAST_OVER_TIME) = range(12)
# hg_topk_order: the direction of scan_range_function_topk
HG_TOPK, HG_BOTTOMK = 0, 1

STATUS = {0: "OK", 1: "INVALID", 2: "UNSUPPORTED", 3: "CUDA", 4: "FORMAT", 5: "OOM", 6: "NOT_FOUND", 7: "INTERNAL"}


class HgError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"HG_ERR_{STATUS.get(code, code)}: {msg}")
        self.code = code


class HgSchemaDesc(C.Structure):
    _fields_ = [("num_columns", C.c_uint32), ("num_primary_keys", C.c_uint32), ("update_mode", C.c_uint32),
                ("_pad", C.c_uint32), ("types", C.POINTER(C.c_uint32)), ("names", C.POINTER(C.c_char_p))]


class HgConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("batch_size", C.c_uint32), ("hbm_budget_bytes", C.c_uint64),
                ("flags", C.c_uint32), ("_pad", C.c_uint32)]


class HgSstDesc(C.Structure):
    _fields_ = [("id", C.c_uint64), ("data", C.c_void_p), ("size", C.c_uint64), ("path", C.c_char_p),
                ("num_rows", C.c_uint32), ("_pad", C.c_uint32), ("time_start", C.c_int64), ("time_end", C.c_int64),
                ("max_sequence", C.c_uint64)]


class HgBytes(C.Structure):
    _fields_ = [("data", C.c_void_p), ("len", C.c_uint64)]


class _HgPredicateLiterals(C.Union):
    _fields_ = [("in_values", C.POINTER(C.c_uint64)), ("in_bytes", C.POINTER(HgBytes))]


class HgPredicate(C.Structure):
    _anonymous_ = ("_lits",)
    _fields_ = [("column", C.c_uint32), ("op", C.c_uint32), ("i64", C.c_int64), ("u64", C.c_uint64), ("f64", C.c_double),
                ("_lits", _HgPredicateLiterals), ("in_count", C.c_uint32), ("_pad", C.c_uint32)]


HG_MAX_BINARY_LITERAL = 65536
_BYTES_LIKE = (bytes, bytearray, memoryview)


def _binary_literals(name: str, lits, keep: list):
    """bytes / bytearray / memoryview literals -> (HgBytes array, count); the buffers are kept alive in `keep`."""
    arr = (HgBytes * max(len(lits), 1))()
    for j, v in enumerate(lits):
        if not isinstance(v, _BYTES_LIKE):
            raise HgError(1, f"literal {v!r} for Binary column {name}: expected bytes, bytearray or memoryview")
        b = bytes(v)
        if b:
            buf = C.create_string_buffer(b, len(b))
            keep.append(buf)
            arr[j].data = C.addressof(buf)
        arr[j].len = len(b)
    keep.append(arr)
    return arr, len(lits)


class HgAggSpec(C.Structure):
    _fields_ = [("group_col", C.c_int32), ("ts_col", C.c_int32), ("window_ms", C.c_int64), ("value_col", C.c_int32),
                ("mode", C.c_uint32)]


class HgScanStats(C.Structure):
    _fields_ = [("rows_in_files", C.c_uint64), ("rows_decoded", C.c_uint64), ("rows_filtered", C.c_uint64),
                ("rows_out", C.c_uint64), ("groups_out", C.c_uint64), ("bytes_h2d", C.c_uint64), ("bytes_d2h", C.c_uint64),
                ("kernel_launches", C.c_uint32), ("path", C.c_uint32), ("gpu_ms", C.c_float), ("kernel_ms", C.c_float), ("merge_ms", C.c_float), ("decomp_ms", C.c_float),
                ("rows_materialized", C.c_uint64)]


class HgAggDevice(C.Structure):
    _fields_ = [("num_groups", C.c_uint64), ("d_gkey", C.c_void_p), ("d_bucket", C.c_void_p), ("d_count", C.c_void_p),
                ("d_sum", C.c_void_p), ("d_min", C.c_void_p), ("d_max", C.c_void_p)]


class HgGroupMap(C.Structure):
    _fields_ = [("keys", C.POINTER(C.c_uint64)), ("groups", C.POINTER(C.c_uint32)), ("count", C.c_uint32), ("_pad", C.c_uint32)]


class HgRangeSpec(C.Structure):
    _fields_ = [("start_ms", C.c_int64), ("end_ms", C.c_int64), ("step_ms", C.c_int64), ("range_ms", C.c_int64)]


class HgColumnWriteOpts(C.Structure):
    _fields_ = [("encoding", C.c_uint8), ("dictionary", C.c_uint8), ("codec", C.c_uint8), ("bloom_filter", C.c_uint8)]


class HgWriteProps(C.Structure):
    _fields_ = [("max_row_group_size", C.c_uint32), ("compression", C.c_uint32), ("enable_sorting_columns", C.c_uint32),
                ("bloom_filter_bytes", C.c_uint32), ("columns", C.POINTER(HgColumnWriteOpts))]


CODECS = {"none": 0, "uncompressed": 0, "snappy": 1, "zstd": 6}
ENCODINGS = {"PLAIN": 0, "RLE": 3, "DELTA_BINARY_PACKED": 5, "DELTA_LENGTH_BYTE_ARRAY": 6, "DELTA_BYTE_ARRAY": 7, "RLE_DICTIONARY": 8}


def _write_props(max_row_group_size: int, compression: str, enable_sorting_columns: bool, columns, bloom_filters=None,
                 bloom_filter_bytes: int = 0) -> HgWriteProps:
    """`columns`: None, or one (encoding, dictionary, codec) per schema column (builtins included), e.g. ("DELTA_BINARY_PACKED", False, "snappy");
    the names map as CODECS / ENCODINGS do, an unknown name becomes a code the library refuses (naming the column).
    `bloom_filters`: None, or one flag per schema column (`config.resolve_bloom_filters`); with `columns` None the other options stay
    PLAIN / no dictionary / `compression`."""
    # with per-column options the table-wide codec is not used (one it cannot name stays harmless)
    codec = CODECS[compression.lower()] if columns is None else CODECS.get(compression.lower(), 0)
    props = HgWriteProps(max_row_group_size, codec, int(enable_sorting_columns), int(bloom_filter_bytes))
    if columns is None and bloom_filters is not None:
        columns = [(0, False, codec)] * len(bloom_filters)
    if columns is not None:
        arr = (HgColumnWriteOpts * max(len(columns), 1))()
        for i, (enc, dictionary, codec) in enumerate(columns):
            arr[i].encoding = enc if isinstance(enc, int) else ENCODINGS.get(str(enc).upper(), 0xFF)
            arr[i].dictionary = int(bool(dictionary))
            arr[i].codec = codec if isinstance(codec, int) else CODECS.get(str(codec).lower(), 0xFF)
            if bloom_filters is not None:
                bf = bloom_filters[i]
                arr[i].bloom_filter = bf if isinstance(bf, int) and not isinstance(bf, bool) else int(bool(bf))
        props.columns = arr
        props._keep = arr
    return props


class HgParquetBloom(C.Structure):
    _fields_ = [("offset", C.c_int64), ("length", C.c_int32), ("num_bytes", C.c_uint32), ("bitset_offset", C.c_uint64),
                ("usable", C.c_uint32), ("_pad", C.c_uint32)]


class HgFileMeta(C.Structure):
    _fields_ = [("size", C.c_uint64), ("num_rows", C.c_uint32), ("_pad", C.c_uint32), ("time_start", C.c_int64), ("time_end", C.c_int64),
                ("max_sequence", C.c_uint64)]


class HgAggCombined(C.Structure):
    _fields_ = [("capacity", C.c_uint64), ("world", C.c_uint32), ("_pad", C.c_uint32), ("d_blocks", C.c_void_p), ("num_groups", C.c_uint64),
                ("reduced_capacity", C.c_uint64), ("d_reduced", C.c_void_p)]


HG_COMBINE_GATHER, HG_COMBINE_REDUCE = 0, 1


class ArrowArrayStream(C.Structure):
    _fields_ = [("get_schema", C.c_void_p), ("get_next", C.c_void_p), ("get_last_error", C.c_void_p),
                ("release", C.c_void_p), ("private_data", C.c_void_p)]


class HgParquetSummary(C.Structure):
    _fields_ = [("num_rows", C.c_uint64), ("num_row_groups", C.c_uint32), ("num_columns", C.c_uint32), ("num_data_pages", C.c_uint64),
                ("sum_page_values", C.c_uint64), ("sum_uncompressed_bytes", C.c_uint64), ("sum_compressed_bytes", C.c_uint64),
                ("codec_mask", C.c_uint32), ("max_pages_per_chunk", C.c_uint32)]


class HgParquetChunk(C.Structure):
    _fields_ = [("num_rows", C.c_uint64), ("num_values", C.c_uint64), ("data_page_offset", C.c_int64), ("total_compressed_size", C.c_int64),
                ("null_count", C.c_int64), ("min", C.c_uint8 * 8), ("max", C.c_uint8 * 8), ("has_min_max", C.c_uint32),
                ("physical_type", C.c_uint32), ("codec", C.c_uint32), ("num_pages", C.c_uint32), ("first_page_payload_offset", C.c_uint64),
                ("first_page_num_values", C.c_uint32), ("first_page_type", C.c_uint32)]


EXPORTS = ["hg_abi_version", "hg_last_error", "hg_engine_create", "hg_engine_destroy", "hg_engine_stream", "hg_engine_set_flags", "hg_sst_load",
           "hg_sst_unload", "hg_sst_resident_bytes", "hg_scan_open", "hg_compact_open", "hg_scan_aggregate",
           "hg_scan_counter_aggregate", "hg_scan_quantile_aggregate", "hg_scan_aggregate_by_map", "hg_scan_aggregate_by_map_device",
           "hg_scan_quantile_aggregate_by_map", "hg_scan_range_aggregate", "hg_scan_range_quantile_aggregate", "hg_scan_range_function",
           "hg_scan_range_function_by_map", "hg_scan_histogram_quantile", "hg_scan_range_function_topk", "hg_scan_aggregate_device", "hg_agg_export_packed", "hg_last_stats", "hg_parquet_inspect", "hg_parquet_chunk_info", "hg_plan_row_groups",
           "hg_parquet_bloom_info", "hg_parquet_bloom_probe",
           "hg_compact_to_sst", "hg_write_batch", "hg_plan_pk_splitters", "hg_comm_unique_id", "hg_comm_init", "hg_comm_destroy", "hg_agg_combine", "hg_comm_sync"]

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(horaedb_b200 has no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.hg_abi_version.restype = C.c_uint32
        L.hg_last_error.restype = C.c_char_p
        L.hg_engine_stream.restype = C.c_void_p
        L.hg_engine_stream.argtypes = [C.c_void_p]
        L.hg_engine_set_flags.argtypes = [C.c_void_p, C.c_uint32]
        L.hg_engine_destroy.argtypes = [C.c_void_p]
        L.hg_engine_destroy.restype = None
        L.hg_comm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.hg_comm_destroy.argtypes = [C.c_void_p]
        L.hg_comm_sync.argtypes = [C.c_void_p]
        L.hg_agg_combine.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p]
        _lib = L
    return _lib


def _check(rc: int):
    if rc != 0:
        raise HgError(rc, lib().hg_last_error().decode())


@dataclass
class SstInput:
    """`SstFile` + `FileMeta` (sst.rs:51-53, 155-160) as passed across the ABI."""
    id: int
    data: Optional[object] = None   # bytes / numpy uint8 / None when resident
    path: Optional[str] = None
    num_rows: int = 0
    time_start: int = 0
    time_end: int = 0
    max_sequence: int = 0
    ptr: int = 0                    # raw host pointer (e.g. pinned memory) used instead of `data`
    size: int = 0


class DeviceArray:
    """Zero-copy view of an engine-owned device buffer (`__cuda_array_interface__`), e.g. for torch.as_tensor(...)."""

    def __init__(self, ptr: int, n: int, typestr: str):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": typestr, "data": (int(ptr or 0), False), "version": 2}


class SchemaHandle:
    """Keeps the ctypes arrays behind an hg_schema_desc alive."""

    def __init__(self, arrow_schema: pa.Schema, num_primary_keys: int, update_mode: int = 0):
        n = len(arrow_schema)
        self.types = (C.c_uint32 * n)(*[HG_TYPES[f.type] if f.type in HG_TYPES else 0xFFFF for f in arrow_schema])
        self.names = (C.c_char_p * n)(*[f.name.encode() for f in arrow_schema])
        self.desc = HgSchemaDesc(n, num_primary_keys, update_mode, 0, self.types, self.names)
        self.arrow_schema = arrow_schema


def _in_set_values(name: str, values) -> np.ndarray:
    """The values of an "in_set" predicate as a contiguous uint64 array in the column's widened domain (two's complement): a numpy
    integer array is converted by numpy (a million ids cost milliseconds), anything else goes through a Python list."""
    if not isinstance(values, np.ndarray):
        vals = list(values)
        for v in vals:
            if isinstance(v, float) and not v.is_integer() or isinstance(v, _BYTES_LIKE):
                raise HgError(1, f"IN_SET literal {v!r} is not an integer for column {name}")
        values = np.array([int(v) & 0xFFFFFFFFFFFFFFFF for v in vals], dtype=np.uint64)
    if values.ndim != 1 or values.dtype.kind not in "iu":
        raise HgError(1, f"IN_SET for column {name}: expected a one-dimensional integer array, got {values.dtype} with shape {values.shape}")
    if values.dtype.kind == "i":
        values = values.astype(np.int64).view(np.uint64)
    return np.ascontiguousarray(values, dtype=np.uint64)


def _group_map(arrow_schema: pa.Schema, group_col: int, keys, groups) -> HgGroupMap:
    """An hg_group_map over numpy copies of `keys` (the key column's widened domain, as for "in_set") and `groups` (u32 ordinals); the
    arrays are kept alive by the returned struct."""
    name = arrow_schema.field(group_col).name if 0 <= group_col < len(arrow_schema) else str(group_col)
    k = _in_set_values(name, keys)
    g = np.asarray(groups)
    if g.ndim != 1 or (g.size and g.dtype.kind not in "iu"):
        raise HgError(1, f"group map for column {name}: groups must be a one-dimensional integer array")
    if g.size and (int(g.min()) < 0 or int(g.max()) > 0xFFFFFFFF):
        raise HgError(1, f"group map for column {name}: a group ordinal outside the u32 range")
    if len(g) != len(k):
        raise HgError(1, f"group map for column {name}: {len(k)} keys but {len(g)} groups")
    g = np.ascontiguousarray(g, dtype=np.uint32)
    m = HgGroupMap(C.cast(C.c_void_p(k.ctypes.data), C.POINTER(C.c_uint64)), C.cast(C.c_void_p(g.ctypes.data), C.POINTER(C.c_uint32)),
                   min(len(k), 0xFFFFFFFF), 0)
    m._keep = (k, g)
    return m


def _quantile_args(quantiles: Sequence[float]):
    """The quantile list of a quantile call: the f64 array (never empty) and its length."""
    return (C.c_double * max(1, len(quantiles)))(*quantiles), C.c_uint32(len(quantiles))


def _make_preds(arrow_schema: pa.Schema, preds: Sequence[tuple]):
    arr = (HgPredicate * max(len(preds), 1))()
    keep = []
    for k, (col, op, lit) in enumerate(preds):
        idx = col if isinstance(col, int) else arrow_schema.get_field_index(col)
        t = arrow_schema.field(idx).type
        arr[k].column = idx
        arr[k].op = HG_OPS[op]
        if op == "in_set":
            # the library refuses float / Binary columns and oversized sets; the array is kept alive for the call
            vals = _in_set_values(arrow_schema.field(idx).name, lit)
            keep.append(vals)
            arr[k].in_values = C.cast(C.c_void_p(vals.ctypes.data), C.POINTER(C.c_uint64))
            arr[k].in_count = min(len(vals), 0xFFFFFFFF)
        elif pa.types.is_binary(t):
            # Binary columns: every operator reads its literal(s) from in_bytes (one for a comparison, the list for "in")
            if op == "in":
                if isinstance(lit, _BYTES_LIKE) or not hasattr(lit, "__iter__"):
                    raise HgError(1, f"IN list for Binary column {arrow_schema.field(idx).name} must be a list of bytes, got {lit!r}")
                lits = list(lit)
            else:
                lits = [lit]
            arr[k].in_bytes, arr[k].in_count = _binary_literals(arrow_schema.field(idx).name, lits, keep)
        elif op == "in":
            bits = []
            for v in lit:
                if pa.types.is_floating(t):
                    bits.append(int(np.array([float(v)], dtype=np.float64).view(np.uint64)[0]))
                else:
                    if isinstance(v, float) and not v.is_integer():
                        raise HgError(1, f"IN literal {v!r} is not integral for column {arrow_schema.field(idx).name}")
                    bits.append(int(v) & 0xFFFFFFFFFFFFFFFF)
            vals = (C.c_uint64 * max(len(bits), 1))(*bits)
            keep.append(vals)
            arr[k].in_values = vals
            arr[k].in_count = len(bits)
        elif pa.types.is_floating(t):
            arr[k].f64 = float(lit)
        else:
            # no silent truncation / wrap-around: a literal the column type cannot hold must be rewritten by the caller
            # (DataFusion would coerce the comparison to a wider type; this ABI compares in the column's own domain)
            if isinstance(lit, float) and not lit.is_integer():
                raise HgError(1, f"predicate literal {lit!r} is not integral for column {arrow_schema.field(idx).name}")
            if not pa.types.is_integer(t):
                raise HgError(2, f"predicates on {t} column {arrow_schema.field(idx).name} are not implemented on the GPU path")
            iv = int(lit)
            bits = t.bit_width
            lo, hi = (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if pa.types.is_signed_integer(t) else (0, (1 << bits) - 1)
            if not lo <= iv <= hi:
                raise HgError(1, f"predicate literal {iv} does not fit column {arrow_schema.field(idx).name} ({t})")
            if pa.types.is_signed_integer(t):
                arr[k].i64 = iv
            else:
                arr[k].u64 = iv
    arr._keep = keep              # IN lists must outlive the call
    return arr


def _check_columns(schema: "SchemaHandle", columns):
    if columns is not None and len(columns) != len(schema.arrow_schema):
        raise HgError(1, f"{len(columns)} column write options for a schema of {len(schema.arrow_schema)} columns")
    return columns


def _check_blooms(schema: "SchemaHandle", bloom_filters):
    if bloom_filters is not None and len(bloom_filters) != len(schema.arrow_schema):
        raise HgError(1, f"{len(bloom_filters)} bloom filter flags for a schema of {len(schema.arrow_schema)} columns")
    return bloom_filters


class Engine:
    """One engine per GPU (per rank).  Thin object wrapper over the C ABI."""

    def __init__(self, device: int = 0, batch_size: int = 8192, hbm_budget_bytes: int = 0, flags: int = 0):
        self._L = lib()
        self._h = C.c_void_p()
        cfg = HgConfig(device, batch_size, hbm_budget_bytes, flags, 0)
        _check(self._L.hg_engine_create(C.byref(cfg), C.byref(self._h)))
        self._keep = []
        self._stats_buf = HgScanStats()

    def close(self):
        if self._h:
            self._L.hg_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def stream_ptr(self) -> int:
        return self._L.hg_engine_stream(self._h)

    def set_flags(self, flags: int) -> None:
        _check(self._L.hg_engine_set_flags(self._h, flags))

    # -- residency
    def _descs(self, ssts: Sequence[SstInput]):
        arr = (HgSstDesc * max(len(ssts), 1))()
        keep = []
        for i, s in enumerate(ssts):
            arr[i].id = s.id
            if s.ptr:
                arr[i].data = s.ptr
                arr[i].size = s.size
            elif s.data is not None:
                buf = np.frombuffer(s.data, dtype=np.uint8) if not isinstance(s.data, np.ndarray) else s.data
                keep.append(buf)
                arr[i].data = buf.ctypes.data
                arr[i].size = buf.nbytes
            else:
                arr[i].data = None
                arr[i].size = 0
            arr[i].path = s.path.encode() if s.path else None
            arr[i].num_rows = s.num_rows
            arr[i].time_start = s.time_start
            arr[i].time_end = s.time_end
            arr[i].max_sequence = s.max_sequence
        return arr, keep

    def load_sst(self, schema: SchemaHandle, sst: SstInput):
        arr, keep = self._descs([sst])
        _check(self._L.hg_sst_load(self._h, C.byref(schema.desc), C.byref(arr[0])))

    def unload_sst(self, id: int):
        _check(self._L.hg_sst_unload(self._h, C.c_uint64(id)))

    def resident_bytes(self) -> int:
        out = C.c_uint64()
        _check(self._L.hg_sst_resident_bytes(self._h, C.byref(out)))
        return out.value

    # -- scan / compaction
    def scan(self, schema: SchemaHandle, ssts: Sequence[SstInput], preds: Sequence[tuple] = (),
             projection: Optional[Sequence[int]] = None, keep_builtin: bool = False) -> pa.RecordBatchReader:
        arr, keep = self._descs(ssts)
        p = _make_preds(schema.arrow_schema, preds)
        proj = (C.c_uint32 * max(len(projection), 1))(*projection) if projection is not None else None
        stream = ArrowArrayStream()
        _check(self._L.hg_scan_open(self._h, C.byref(schema.desc), arr, C.c_size_t(len(ssts)), p, C.c_size_t(len(preds)),
                                    proj, C.c_size_t(len(projection) if projection is not None else 0), int(keep_builtin),
                                    C.byref(stream)))
        return pa.RecordBatchReader._import_from_c(C.addressof(stream))

    def compact(self, schema: SchemaHandle, ssts: Sequence[SstInput]) -> pa.RecordBatchReader:
        arr, keep = self._descs(ssts)
        stream = ArrowArrayStream()
        _check(self._L.hg_compact_open(self._h, C.byref(schema.desc), arr, C.c_size_t(len(ssts)), C.byref(stream)))
        return pa.RecordBatchReader._import_from_c(C.addressof(stream))

    def compact_to_sst(self, schema: SchemaHandle, ssts: Sequence[SstInput], out_path: str, max_row_group_size: int = 8192,
                       compression: str = "snappy", enable_sorting_columns: bool = True, shard_preds: Sequence[tuple] = (),
                       columns: Optional[Sequence[tuple]] = None, bloom_filters: Optional[Sequence[bool]] = None,
                       bloom_filter_bytes: int = 0) -> "HgFileMeta":
        """`Executor::do_compaction` on the GPU end to end: merge + dedup + Parquet encode, written to `out_path`.
        `shard_preds` = this GPU's pk0 range in a multi-GPU compaction (see `plan_pk_splitters`).
        `columns` = per-column writer options, one (encoding, dictionary, codec) per schema column (`config.resolve_column_options`);
        None = PLAIN with `compression` everywhere.  `bloom_filters` = None (no filters) or one flag per schema column
        (`config.resolve_bloom_filters`); `bloom_filter_bytes` = the bitset size of every filter, 0 = 1 MiB (parquet-rs's default)."""
        arr, keep = self._descs(ssts)
        p = _make_preds(schema.arrow_schema, shard_preds)
        props = _write_props(max_row_group_size, compression, enable_sorting_columns, _check_columns(schema, columns),
                             _check_blooms(schema, bloom_filters), bloom_filter_bytes)
        meta = HgFileMeta()
        _check(self._L.hg_compact_to_sst(self._h, C.byref(schema.desc), arr, C.c_size_t(len(ssts)), p, C.c_size_t(len(shard_preds)), C.byref(props),
                                         out_path.encode(), C.byref(meta)))
        return meta

    def write_batch(self, schema: SchemaHandle, batch: pa.RecordBatch, sequence: int, out_path: str, max_row_group_size: int = 8192,
                    compression: str = "snappy", enable_sorting_columns: bool = True, columns: Optional[Sequence[tuple]] = None,
                    bloom_filters: Optional[Sequence[bool]] = None, bloom_filter_bytes: int = 0) -> "HgFileMeta":
        """`ObjectBasedStorage::write_batch` on the GPU (storage.rs:189-225): sort by the primary keys, append the builtin columns,
        encode, write `out_path`.  `batch` holds the USER columns; it travels as an Arrow C struct array.  `columns`, `bloom_filters`,
        `bloom_filter_bytes`: as for `compact_to_sst`, builtin columns included."""
        user = len(schema.arrow_schema) - 2
        if batch.num_columns != user:
            raise HgError(1, f"batch has {batch.num_columns} columns, the schema has {user} user columns")
        cols = [batch.column(i).cast(schema.arrow_schema.field(i).type) for i in range(user)]
        st = pa.StructArray.from_arrays(cols, fields=[schema.arrow_schema.field(i) for i in range(user)])

        class _CArray(C.Structure):
            _fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64), ("n_children", C.c_int64),
                        ("buffers", C.c_void_p), ("children", C.c_void_p), ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]

        carr = _CArray()
        st._export_to_c(C.addressof(carr))
        props = _write_props(max_row_group_size, compression, enable_sorting_columns, _check_columns(schema, columns),
                             _check_blooms(schema, bloom_filters), bloom_filter_bytes)
        meta = HgFileMeta()
        try:
            _check(self._L.hg_write_batch(self._h, C.byref(schema.desc), C.byref(carr), C.c_uint64(sequence), C.byref(props), out_path.encode(), C.byref(meta)))
        finally:
            pa.Array._import_from_c(C.addressof(carr), st.type)      # takes the exported array back: its release callback runs on GC
        return meta

    def _aggregate(self, fn, schema: SchemaHandle, ssts: Sequence[SstInput], preds: Sequence[tuple], spec: tuple, *args, device: bool = False):
        """One aggregate call `fn(engine, schema, ssts, preds, spec, *args, out)` with spec = (group_col, ts_col, window_ms, value_col,
        mode): the result read from its Arrow stream, or its HgAggDevice (device=True)."""
        arr, keep = self._descs(ssts)          # keep holds the SSTs' host buffers until the call has returned
        p = _make_preds(schema.arrow_schema, preds)
        out = HgAggDevice() if device else ArrowArrayStream()
        _check(fn(self._h, C.byref(schema.desc), arr, C.c_size_t(len(ssts)), p, C.c_size_t(len(preds)), C.byref(HgAggSpec(*spec)), *args,
                  C.byref(out)))
        return out if device else pa.RecordBatchReader._import_from_c(C.addressof(out)).read_all()

    def scan_aggregate(self, schema: SchemaHandle, ssts: Sequence[SstInput], preds: Sequence[tuple] = (), group_col: int = 0,
                       ts_col: int = -1, window_ms: int = 0, value_col: int = -1, mode: int = 0) -> pa.Table:
        return self._aggregate(self._L.hg_scan_aggregate, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode))

    def scan_counter_aggregate(self, schema: SchemaHandle, ssts: Sequence[SstInput], preds: Sequence[tuple] = (), group_col: int = 0,
                               ts_col: int = 1, window_ms: int = 0, value_col: int = 2, mode: int = 0) -> pa.Table:
        """Counter partials per (series, bucket): key, [bucket,] count, first_ts, first_value, last_ts, last_value, increase, resets
        (`hg_scan_counter_aggregate`).  first_* / last_* are null for a group without a non-null value."""
        return self._aggregate(self._L.hg_scan_counter_aggregate, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode))

    def scan_quantile_aggregate(self, schema: SchemaHandle, ssts: Sequence[SstInput], preds: Sequence[tuple] = (), group_col: int = 0,
                                ts_col: int = -1, window_ms: int = 0, value_col: int = 2, mode: int = 0,
                                quantiles: Sequence[float] = (0.5,)) -> pa.Table:
        """Exact quantiles per (group, bucket) (`hg_scan_quantile_aggregate`): key, [bucket,] count, quantile_0 .. quantile_(n-1), the
        groups of `scan_aggregate` for the same spec.  Over a group's m non-NULL values v(0) <= ... <= v(m-1) (floats in IEEE totalOrder,
        each converted to f64), for each q: rank = q * (m - 1), lo = floor(rank), hi = min(lo + 1, m - 1), w = rank - lo, and the result
        is v(lo) when w == 0, else v(lo) * (1 - w) + v(hi) * w, every operation rounded to f64 on its own.  NULL when m = 0."""
        return self._aggregate(self._L.hg_scan_quantile_aggregate, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               *_quantile_args(quantiles))

    def scan_aggregate_by_map(self, schema: SchemaHandle, ssts: Sequence[SstInput], keys, groups, preds: Sequence[tuple] = (),
                              group_col: int = 0, ts_col: int = -1, window_ms: int = 0, value_col: int = -1, mode: int = 0) -> pa.Table:
        """count / sum / min / max per (label group, bucket) (`hg_scan_aggregate_by_map`): row r belongs to group groups[i] when its
        `group_col` value is keys[i]; rows whose key is not in `keys` do not take part.  Columns: group (u32), [bucket,] count[, sum, min,
        max], groups sorted by (ordinal, bucket).  keys / groups: integer arrays of one length (numpy arrays pass without a Python loop)."""
        return self._aggregate(self._L.hg_scan_aggregate_by_map, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               C.byref(_group_map(schema.arrow_schema, group_col, keys, groups)))

    def scan_aggregate_by_map_device(self, schema: SchemaHandle, ssts: Sequence[SstInput], keys, groups, preds: Sequence[tuple] = (),
                                     group_col: int = 0, ts_col: int = -1, window_ms: int = 0, value_col: int = -1,
                                     mode: int = 0) -> HgAggDevice:
        """`scan_aggregate_by_map` with its result left on the device (d_gkey: the u32 ordinals), for `export_packed` / `combine`."""
        return self._aggregate(self._L.hg_scan_aggregate_by_map_device, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               C.byref(_group_map(schema.arrow_schema, group_col, keys, groups)), device=True)

    def scan_quantile_aggregate_by_map(self, schema: SchemaHandle, ssts: Sequence[SstInput], keys, groups, preds: Sequence[tuple] = (),
                                       group_col: int = 0, ts_col: int = -1, window_ms: int = 0, value_col: int = 2, mode: int = 0,
                                       quantiles: Sequence[float] = (0.5,)) -> pa.Table:
        """Quantiles per (label group, bucket) (`hg_scan_quantile_aggregate_by_map`): the groups of `scan_aggregate_by_map`, each with
        `scan_quantile_aggregate`'s definition.  Columns: group (u32), [bucket,] count, quantile_0 .. quantile_(n-1)."""
        return self._aggregate(self._L.hg_scan_quantile_aggregate_by_map, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               C.byref(_group_map(schema.arrow_schema, group_col, keys, groups)), *_quantile_args(quantiles))

    def scan_range_aggregate(self, schema: SchemaHandle, ssts: Sequence[SstInput], preds: Sequence[tuple] = (), start_ms: int = 0,
                             end_ms: int = 0, step_ms: int = 1, range_ms: int = 1, value_col: int = 2, mode: int = 0, group_col: int = 0,
                             ts_col: int = 1, window_ms: int = 0) -> pa.Table:
        """Range windows per series (`hg_scan_range_aggregate`): at t = start_ms, start_ms + step_ms, .. <= end_ms, the series' rows with
        t - range_ms < ts <= t.  Columns: series key, t, count, sum, min, max, first_ts, first_value, last_ts, last_value, increase, resets;
        a window appears iff it has a row; first_* / last_* are null for a window without a non-null value.  group_col / ts_col /
        window_ms keep their defaults (the series, the time column, no buckets): the library refuses any other shape."""
        return self._aggregate(self._L.hg_scan_range_aggregate, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               C.byref(HgRangeSpec(start_ms, end_ms, step_ms, range_ms)))

    def scan_range_quantile_aggregate(self, schema: SchemaHandle, ssts: Sequence[SstInput], preds: Sequence[tuple] = (), start_ms: int = 0,
                                      end_ms: int = 0, step_ms: int = 1, range_ms: int = 1, value_col: int = 2, mode: int = 0,
                                      quantiles: Sequence[float] = (0.5,), group_col: int = 0, ts_col: int = 1, window_ms: int = 0) -> pa.Table:
        """Quantiles over range windows (`hg_scan_range_quantile_aggregate`): the windows of `scan_range_aggregate`, each with
        `scan_quantile_aggregate`'s definition.  Columns: series key, t, count, quantile_0 .. quantile_(n-1)."""
        return self._aggregate(self._L.hg_scan_range_quantile_aggregate, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               C.byref(HgRangeSpec(start_ms, end_ms, step_ms, range_ms)), *_quantile_args(quantiles))

    def scan_range_function(self, schema: SchemaHandle, ssts: Sequence[SstInput], fn: int, preds: Sequence[tuple] = (), start_ms: int = 0,
                            end_ms: int = 0, step_ms: int = 1, range_ms: int = 1, value_col: int = 2, mode: int = 0, group_col: int = 0,
                            ts_col: int = 1, window_ms: int = 0) -> pa.Table:
        """A PromQL range function per series and step (`hg_scan_range_function`): fn (HG_FN_*) over the windows of
        `scan_range_aggregate`.  Columns: series key, t, value; a row appears iff its window has a value (rate needs two samples, ...)."""
        return self._aggregate(self._L.hg_scan_range_function, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               C.byref(HgRangeSpec(start_ms, end_ms, step_ms, range_ms)), C.c_uint32(fn))

    def scan_range_function_by_map(self, schema: SchemaHandle, ssts: Sequence[SstInput], fn: int, keys, groups, preds: Sequence[tuple] = (),
                                   start_ms: int = 0, end_ms: int = 0, step_ms: int = 1, range_ms: int = 1, value_col: int = 2, mode: int = 0,
                                   group_col: int = 0, ts_col: int = 1, window_ms: int = 0) -> pa.Table:
        """`scan_range_function` aggregated across series by label group (`hg_scan_range_function_by_map`): series keys[i] belongs to
        group groups[i]; per (group, t) the count / sum / min / max of the values of its series that have one.  Columns: group (u32), t,
        count, sum, min, max, sorted by (ordinal, t)."""
        return self._aggregate(self._L.hg_scan_range_function_by_map, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               C.byref(HgRangeSpec(start_ms, end_ms, step_ms, range_ms)), C.c_uint32(fn),
                               C.byref(_group_map(schema.arrow_schema, group_col, keys, groups)))

    def scan_range_function_topk(self, schema: SchemaHandle, ssts: Sequence[SstInput], fn: int, k: int, keys, groups, preds: Sequence[tuple] = (),
                                 start_ms: int = 0, end_ms: int = 0, step_ms: int = 1, range_ms: int = 1, order: int = HG_TOPK, value_col: int = 2,
                                 mode: int = 0, group_col: int = 0, ts_col: int = 1, window_ms: int = 0) -> pa.Table:
        """topk / bottomk(k, fn(x[r])) by label group (`hg_scan_range_function_topk`): the series and values of `scan_range_function_by_map`
        per (group, t), ordered by value (descending for HG_TOPK, ascending for HG_BOTTOMK; NaN last in both, ties in series-key order),
        the first k of each.  Columns: group (u32), t, series key, value, sorted by (ordinal, t, rank)."""
        return self._aggregate(self._L.hg_scan_range_function_topk, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               C.byref(HgRangeSpec(start_ms, end_ms, step_ms, range_ms)), C.c_uint32(fn),
                               C.byref(_group_map(schema.arrow_schema, group_col, keys, groups)), C.c_uint32(k), C.c_uint32(order))

    def scan_histogram_quantile(self, schema: SchemaHandle, ssts: Sequence[SstInput], fn: int, keys, groups, upper_bounds,
                                quantiles: Sequence[float], preds: Sequence[tuple] = (), start_ms: int = 0, end_ms: int = 0, step_ms: int = 1,
                                range_ms: int = 1, value_col: int = 2, mode: int = 0, group_col: int = 0, ts_col: int = 1,
                                window_ms: int = 0) -> pa.Table:
        """histogram_quantile(q, sum by (..., le) (fn(x[r]))) per label group and step (`hg_scan_histogram_quantile`): series keys[i] is
        the bucket of group groups[i] with upper bound upper_bounds[i] (its `le` as a float).  The bucket counts are
        `scan_range_function_by_map`'s sums per (group, bound); per (group, t) with a bucket, Prometheus's bucketQuantile of each q.
        Columns: group (u32), t, forced_monotonic (u8), quantile_0 .. quantile_(n-1), sorted by (ordinal, t)."""
        m = _group_map(schema.arrow_schema, group_col, keys, groups)
        b = np.ascontiguousarray(np.asarray(upper_bounds, dtype=np.float64))
        if b.ndim != 1 or len(b) != m.count:
            raise HgError(1, f"histogram map: {m.count} keys but {b.size} upper bounds")
        return self._aggregate(self._L.hg_scan_histogram_quantile, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode),
                               C.byref(HgRangeSpec(start_ms, end_ms, step_ms, range_ms)), C.c_uint32(fn), C.byref(m),
                               C.cast(C.c_void_p(b.ctypes.data), C.POINTER(C.c_double)), *_quantile_args(quantiles))

    def scan_aggregate_device(self, schema: SchemaHandle, ssts: Sequence[SstInput], preds: Sequence[tuple] = (),
                              group_col: int = 0, ts_col: int = -1, window_ms: int = 0, value_col: int = -1, mode: int = 0) -> HgAggDevice:
        return self._aggregate(self._L.hg_scan_aggregate_device, schema, ssts, preds, (group_col, ts_col, window_ms, value_col, mode), device=True)

    def prepare_aggregate(self, schema: SchemaHandle, ssts: Sequence[SstInput], preds: Sequence[tuple] = (), group_col: int = 0,
                          ts_col: int = -1, window_ms: int = 0, value_col: int = -1, mode: int = 0) -> "PreparedAggregate":
        """Marshal the arguments of `scan_aggregate_device` once; `run()` is then a single C call (what a compiled host pays)."""
        return PreparedAggregate(self, schema, ssts, preds, group_col, ts_col, window_ms, value_col, mode)

    def stats_struct(self) -> "HgScanStats":
        """hg_last_stats into a reused ctypes struct (no dict): for tight measurement loops."""
        _check(self._L.hg_last_stats(self._h, C.byref(self._stats_buf)))
        return self._stats_buf

    def export_packed(self, d_dst: int, cap: int) -> None:
        """Pack the last device aggregate into a caller-owned [6, cap] int64 device buffer (engine stream)."""
        _check(self._L.hg_agg_export_packed(self._h, C.c_void_p(d_dst), C.c_uint64(cap)))

    # -- multi-GPU combine (comm.cu): the NCCL id travels over the host's own channel (here: torch.distributed)
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        _check(lib().hg_comm_unique_id(buf))
        return bytes(buf)

    def comm_init(self, uid: bytes, rank: int, world: int) -> None:
        buf = (C.c_uint8 * 128)(*uid)
        _check(self._L.hg_comm_init(self._h, buf, rank, world))

    def comm_destroy(self) -> None:
        _check(self._L.hg_comm_destroy(self._h))

    def combine(self, mode: int = 0, capacity_hint: int = 0) -> "HgAggCombined":
        out = HgAggCombined()
        _check(self._L.hg_agg_combine(self._h, C.c_uint32(mode), C.c_uint64(capacity_hint), C.byref(out)))
        return out

    def comm_sync(self) -> None:
        _check(self._L.hg_comm_sync(self._h))

    def stats(self) -> dict:
        st = HgScanStats()
        _check(self._L.hg_last_stats(self._h, C.byref(st)))
        return {f[0]: getattr(st, f[0]) for f in HgScanStats._fields_ if not f[0].startswith("_")}


class PreparedAggregate:
    """The ctypes argument block of one `hg_scan_aggregate_device` call, built once and reused."""

    def __init__(self, eng: Engine, schema: SchemaHandle, ssts, preds, group_col, ts_col, window_ms, value_col, mode=0):
        self._eng = eng
        self._schema = schema
        self._arr, self._keep = eng._descs(ssts)
        self._p = _make_preds(schema.arrow_schema, preds)
        self._spec = HgAggSpec(group_col, ts_col, window_ms, value_col, mode)
        self.out = HgAggDevice()
        self._fn = eng._L.hg_scan_aggregate_device
        self._args = (eng._h, C.byref(schema.desc), self._arr, C.c_size_t(len(ssts)), self._p, C.c_size_t(len(preds)),
                      C.byref(self._spec), C.byref(self.out))

    def run(self) -> HgAggDevice:
        rc = self._fn(*self._args)
        if rc:
            _check(rc)
        return self.out


def parquet_inspect(data: bytes) -> dict:
    """Host-only (no GPU): the library's reading of an SST's footer and page headers."""
    L = lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    out = HgParquetSummary()
    _check(L.hg_parquet_inspect(C.c_void_p(buf.ctypes.data), C.c_uint64(buf.nbytes), C.byref(out)))
    return {f[0]: getattr(out, f[0]) for f in HgParquetSummary._fields_}


def parquet_chunk_info(data: bytes, row_group: int, column: int) -> dict:
    L = lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    out = HgParquetChunk()
    _check(L.hg_parquet_chunk_info(C.c_void_p(buf.ctypes.data), C.c_uint64(buf.nbytes), C.c_uint32(row_group), C.c_uint32(column), C.byref(out)))
    d = {f[0]: getattr(out, f[0]) for f in HgParquetChunk._fields_}
    d["min"], d["max"] = bytes(out.min), bytes(out.max)
    return d


def parquet_bloom_info(data: bytes, row_group: int, column: int) -> dict:
    """Host-only (no GPU): the bloom filter of one column chunk as the planner reads it (`usable` = 0: none, or ignored)."""
    L = lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    out = HgParquetBloom()
    _check(L.hg_parquet_bloom_info(C.c_void_p(buf.ctypes.data), C.c_uint64(buf.nbytes), C.c_uint32(row_group), C.c_uint32(column), C.byref(out)))
    return {f[0]: getattr(out, f[0]) for f in HgParquetBloom._fields_ if f[0] != "_pad"}


def parquet_bloom_probe(data: bytes, row_group: int, column: int, value: bytes) -> bool:
    """Host-only (no GPU): may the chunk's bloom filter hold the value whose PLAIN bytes (4 or 8) are `value`?  True without a usable filter."""
    L = lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    v = C.create_string_buffer(bytes(value), len(value))
    maybe = C.c_int()
    _check(L.hg_parquet_bloom_probe(C.c_void_p(buf.ctypes.data), C.c_uint64(buf.nbytes), C.c_uint32(row_group), C.c_uint32(column), v,
                                    C.c_uint32(len(value)), C.byref(maybe)))
    return bool(maybe.value)


def plan_pk_splitters(schema: "SchemaHandle", datas: Sequence[bytes], parts: int) -> list:
    """Host-only (no GPU): `parts - 1` pk0 splitters that balance the rows of the inputs (multi-GPU compaction, SURVEY 8e)."""
    L = lib()
    arr = (HgSstDesc * max(len(datas), 1))()
    keep = []
    for i, d in enumerate(datas):
        buf = np.frombuffer(d, dtype=np.uint8)
        keep.append(buf)
        arr[i].id = i
        arr[i].data = buf.ctypes.data
        arr[i].size = buf.nbytes
    out = (C.c_uint64 * max(parts - 1, 1))()
    _check(L.hg_plan_pk_splitters(C.byref(schema.desc), arr, C.c_size_t(len(datas)), C.c_uint32(parts), out))
    t = schema.arrow_schema.field(0).type
    vals = [int(out[i]) for i in range(parts - 1)]
    if pa.types.is_signed_integer(t):
        vals = [v - (1 << 64) if v >= (1 << 63) else v for v in vals]
    return vals


def shard_range_preds(schema: "SchemaHandle", splitters: Sequence[int], rank: int) -> list:
    """The pk0 range of `rank` among len(splitters) + 1 shards, as predicates for `compact_to_sst(shard_preds=...)`."""
    name = schema.arrow_schema.field(0).name
    preds = []
    if rank > 0:
        preds.append((name, "ge", splitters[rank - 1]))
    if rank < len(splitters):
        preds.append((name, "lt", splitters[rank]))
    return preds


def plan_row_groups(schema: "SchemaHandle", data: bytes, preds: Sequence[tuple] = ()) -> list:
    """Host-only (no GPU): the planner's row-group pruning (statistics, then bloom filters) for one SST -> one 0/1 flag per row group."""
    L = lib()
    buf = np.frombuffer(data, dtype=np.uint8)
    p = _make_preds(schema.arrow_schema, preds)
    cap = 1 << 16
    keep = (C.c_uint8 * cap)()
    n = C.c_uint32()
    _check(L.hg_plan_row_groups(C.byref(schema.desc), C.c_void_p(buf.ctypes.data), C.c_uint64(buf.nbytes), p, C.c_size_t(len(preds)),
                                keep, C.c_uint32(cap), C.byref(n)))
    return [int(keep[i]) for i in range(n.value)]
