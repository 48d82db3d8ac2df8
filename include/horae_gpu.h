/*
 * horae_gpu.h — C ABI of libhorae_gpu.so, the H100 (sm_90a) implementation of HoraeDB's columnar hot path.
 *
 * Every entry point replaces one seam of the reference (paths relative to apache/horaedb @ 9cec5636,
 * src/columnar_storage/src/):
 *
 *   hg_scan_open         ParquetReader::build_df_plan(ssts, projection, predicates, keep_builtin=false)
 *                        + execute_stream                      read.rs:429-494, storage.rs:350-369
 *                        i.e. ParquetExec -> FilterExec -> SortPreservingMergeExec -> MergeExec(LastValue)
 *   hg_compact_open      the same plan as built by Executor::do_compaction: no predicate, keep_builtin=true
 *                                                              compaction/executor.rs:164-171
 *   hg_scan_aggregate*   the time-bucket aggregation the metric engine is meant to run on top of the scan
 *                        (absent in the reference: metric_engine/src/metric/mod.rs:37-49 is todo!();
 *                        window arithmetic = Timestamp::truncate_by, types.rs:82-85)
 *   hg_scan_counter_aggregate   the same buckets with counter partials: first / last sample, increase, resets
 *   hg_scan_quantile_aggregate  the same groups and buckets with exact, interpolated quantiles of a value column
 *   hg_scan_aggregate_by_map    count / sum / min / max and quantiles per caller-given label group (a series -> group map) and bucket
 *   hg_sst_load/unload   residency of immutable SST bytes in HBM, keyed by FileId (sst.rs:48, 193-205)
 *   hg_schema_desc       StorageSchema (types.rs:143-157);   hg_sst_desc = SstFile + FileMeta (sst.rs:51-53,155-160)
 *   hg_predicate         the lowered form of ScanRequest.predicate: Vec<Expr> (storage.rs:65-70) — a conjunction of
 *                        `column <op> literal`; anything else must be rejected by the caller (no CPU fallback)
 *
 * Results travel as Arrow C streams (arrow_c_abi.h): the Rust shim wraps them with
 * arrow::ffi_stream::ArrowArrayStreamReader and hands the batches to DataFusion (see INTEGRATION.md).
 *
 * Conventions: plain C types only; every function returns an hg_status (0 = OK) and records a message readable with
 * hg_last_error() on the calling thread; nothing throws or aborts across the boundary.  The engine handle is
 * thread-safe (calls are serialised per engine); streams may be consumed from any thread.
 */
#ifndef HORAE_GPU_H
#define HORAE_GPU_H

#include <stddef.h>
#include <stdint.h>

#include "arrow_c_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The version of the layouts and calls below.  hg_scan_counter_aggregate, hg_scan_quantile_aggregate, hg_scan_aggregate_by_map,
 * hg_scan_aggregate_by_map_device and hg_scan_quantile_aggregate_by_map came later than the rest of version 8: a caller that must also
 * run against an older version-8 library resolves them at run time (dlsym) or binds at load (-Wl,-z,now), so that their absence is
 * found before the first call. */
#define HG_ABI_VERSION 8u

typedef struct hg_engine hg_engine;

typedef enum {
  HG_OK = 0,
  HG_ERR_INVALID = 1,      /* bad argument / schema mismatch                       (ensure!, macros.rs:36-52) */
  HG_ERR_UNSUPPORTED = 2,  /* encoding / codec / type / expression not implemented on the GPU path (never a CPU fallback) */
  HG_ERR_CUDA = 3,
  HG_ERR_FORMAT = 4,       /* malformed Parquet: footer / page headers, or page contents found inconsistent on the device (levels, dictionary
                              indices, compressed streams, rows that contradict their chunk statistics or the file's sort order) */
  HG_ERR_OOM = 5,          /* HBM admission control (the analogue of Executor::pre_check, executor.rs:93-114) */
  HG_ERR_NOT_FOUND = 6,
  HG_ERR_INTERNAL = 7
} hg_status;

/* Arrow primitive types the reference's primary_key_eq / value columns use (read.rs:269-286) */
typedef enum {
  HG_U8 = 0, HG_I8 = 1, HG_U16 = 2, HG_I16 = 3, HG_U32 = 4, HG_I32 = 5, HG_U64 = 6, HG_I64 = 7, HG_F32 = 8, HG_F64 = 9,
  HG_BINARY = 10   /* Arrow Binary / Parquet BYTE_ARRAY: value columns only (what BytesMergeOperator concatenates, operator.rs:47-111) */
} hg_type;

typedef enum { HG_UPDATE_OVERWRITE = 0, HG_UPDATE_APPEND = 1 } hg_update_mode; /* config.rs:166-172 */

typedef enum { HG_OP_EQ = 0, HG_OP_NE = 1, HG_OP_LT = 2, HG_OP_LE = 3, HG_OP_GT = 4, HG_OP_GE = 5, HG_OP_IN = 6, HG_OP_IN_SET = 7 } hg_op;
#define HG_MAX_IN_LIST 64u
/* HG_OP_IN_SET: `col IN (a large set)` — the series ids an index lookup returned, DataFusion's InList beyond HG_MAX_IN_LIST literals or its
 * InSet.  Same meaning as HG_OP_IN (NULL IN_SET (..) is false; an empty set matches no row), up to HG_MAX_IN_SET values.  Integer columns
 * only (float / Binary column: HG_ERR_UNSUPPORTED); scans and aggregates run on the general pipeline; row groups are pruned by their
 * statistics against the sorted set, bloom filters are not consulted.  Not a shard predicate of hg_compact_to_sst (HG_ERR_INVALID). */
#define HG_MAX_IN_SET (1u << 24)

/* StorageSchema (types.rs:143-157): columns = pk0..pkN-1, values..., __seq__ (u64), __reserved__ (u64) */
typedef struct {
  uint32_t num_columns;       /* including the two builtin columns */
  uint32_t num_primary_keys;
  uint32_t update_mode;       /* hg_update_mode: OVERWRITE = LastValueOperator (operator.rs:37-44); APPEND = BytesMergeOperator
                                 (operator.rs:47-111: every value column must be HG_BINARY; the run's values are concatenated in
                                 (pk, seq) order, the other columns come from the run's FIRST row) */
  uint32_t _pad;
  const uint32_t* types;      /* hg_type per column */
  const char* const* names;   /* column names (for the exported Arrow schema) */
} hg_schema_desc;

typedef struct {
  int32_t device;             /* CUDA ordinal (one engine per GPU / per rank) */
  uint32_t batch_size;        /* DataFusion batch_size the merge re-batches at; 0 = 8192 */
  uint64_t hbm_budget_bytes;  /* 0 = no admission limit */
  uint32_t flags;             /* HG_FLAG_* */
  uint32_t _pad;
} hg_config;

#define HG_FLAG_NO_PRUNING 1u   /* disable row-group pruning by chunk statistics (for A/B measurements) */
#define HG_FLAG_NO_FUSED 2u     /* force the general (materialising) pipeline even when the fused fast path applies */
#define HG_FLAG_NO_LATE_MATERIALIZATION 4u   /* fused path: load every needed column of every row (no predicate gate) */
#define HG_FLAG_PAIRWISE_MERGE 8u   /* k-way merge by log2(k) pairwise passes over 32-byte records even when the packed-key single pass applies (A/B) */
#define HG_FLAG_NO_BLOOM_FILTER 16u /* disable row-group pruning by bloom filters only (A/B); HG_FLAG_NO_PRUNING disables it as well */

/* SstFile + FileMeta (sst.rs:51-53, 155-160).  `data` may be NULL when the file is already resident (hg_sst_load). */
typedef struct {
  uint64_t id;
  const uint8_t* data;        /* whole-file bytes in host memory, or NULL */
  uint64_t size;
  const char* path;           /* optional: "{root}/data/{id}.sst" (sst.rs:202-204), read when data == NULL and not resident */
  uint32_t num_rows;
  uint32_t _pad;
  int64_t time_start, time_end;   /* [start, end) */
  uint64_t max_sequence;
} hg_sst_desc;

/* One byte string (a Binary literal).  data may be NULL only when len == 0. */
typedef struct {
  const uint8_t* data;
  uint64_t len;
} hg_bytes;
#define HG_MAX_BINARY_LITERAL 65536u   /* bytes of one Binary literal, at most */

typedef struct {
  uint32_t column;            /* index into the storage schema */
  uint32_t op;                /* hg_op */
  int64_t i64;                /* literal for signed integer columns */
  uint64_t u64;               /* literal for unsigned integer columns */
  double f64;                 /* literal for float columns */
  union {
    const uint64_t* in_values;  /* HG_OP_IN (`col IN (..)`, DataFusion InListExpr): in_count values in the column's widened domain */
                                /*   (i64 / u64 two's complement, f64 bit patterns); at most HG_MAX_IN_LIST; NULL IN (..) is false */
                                /* HG_OP_IN_SET: the same field, at most HG_MAX_IN_SET values, in any order, duplicates allowed */
    const hg_bytes* in_bytes;   /* HG_BINARY columns, EVERY operator: the literal(s) in_bytes[0 .. in_count), in_count = 1 for the
                                   comparisons, 0 .. HG_MAX_IN_LIST for HG_OP_IN, each at most HG_MAX_BINARY_LITERAL bytes (else
                                   HG_ERR_INVALID).  Binary values order as arrow-rs BinaryArray: unsigned bytes lexicographically, a
                                   proper prefix first (b"" < b"\x00" < b"ab" < b"ab\x00" < b"b").  i64 / u64 / f64 are not read. */
  };
  uint32_t in_count, _pad;
} hg_predicate;

/* GROUP BY (group column, time bucket) over the post-dedup scan output.
 * mode HG_AGG_RUNS: groups are the maximal runs of equal (group value, bucket) in the stream — exact GROUP BY when the key
 *   is a prefix of the sort order (series_id [, ts bucket]); groups come out in stream (key) order.
 * mode HG_AGG_HASH: true GROUP BY for ANY key (e.g. per-(tag, bucket)): radix-partitioned, every group's rows are added in
 *   stream order, groups come out sorted by (group value, bucket).  Identical to RUNS for sort-prefix keys. */
typedef enum { HG_AGG_RUNS = 0, HG_AGG_HASH = 1 } hg_agg_mode;
typedef struct {
  int32_t group_col;          /* -1: one global group */
  int32_t ts_col;             /* -1: no bucketing */
  int64_t window_ms;          /* bucket = ts / window_ms * window_ms (truncating, types.rs:82-85) */
  int32_t value_col;          /* -1: count(*) only */
  uint32_t mode;              /* hg_agg_mode */
} hg_agg_spec;

typedef struct {
  uint64_t rows_in_files;     /* rows of the selected SSTs */
  uint64_t rows_decoded;      /* after row-group pruning */
  uint64_t rows_filtered;     /* after the predicate */
  uint64_t rows_out;          /* after merge + dedup */
  uint64_t groups_out;
  uint64_t bytes_h2d, bytes_d2h;
  uint32_t kernel_launches;   /* kernels launched by the last call */
  uint32_t path;              /* bit 0: 0 = general pipeline, 1 = fused fast path;  bit 1: the call ran twice (a transient load's
                                 compressed page prefix ended before the last needed row: repeated with whole pages) */
  float gpu_ms;               /* device time of the last call, first kernel to last (CUDA events on the engine stream) */
  float kernel_ms;            /* device time of the call's dominant kernel alone (fused scan / page decode) */
  float merge_ms;             /* device time of S4-S6 (sort records, merge passes, dedup, compaction of survivors) */
  float decomp_ms;            /* device time of the page-decompression stage (Snappy; fused path), when one ran */
  uint64_t rows_materialized; /* fused path: rows whose non-gate columns were read (== rows_decoded without the gate);
                                 general pipeline: rows_decoded */
} hg_scan_stats;

/* Device-resident aggregate (for the NCCL combine and HBM-resident timing); valid until the next call on the engine. */
typedef struct {
  uint64_t num_groups;
  const void* d_gkey;         /* group column values, native width */
  const int64_t* d_bucket;
  const uint64_t* d_count;
  const double* d_sum;
  const double* d_min;
  const double* d_max;
} hg_agg_device;

uint32_t hg_abi_version(void);
const char* hg_last_error(void);

int hg_engine_create(const hg_config* cfg, hg_engine** out);
void hg_engine_destroy(hg_engine* e);
void* hg_engine_stream(hg_engine* e); /* the cudaStream_t every kernel of this engine is launched on */
int hg_engine_set_flags(hg_engine* e, uint32_t flags); /* replaces hg_config.flags for the following calls (A/B measurements) */

int hg_sst_load(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* sst);
int hg_sst_unload(hg_engine* e, uint64_t id);
int hg_sst_resident_bytes(hg_engine* e, uint64_t* out);

int hg_scan_open(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                 const hg_predicate* preds, size_t n_preds, const uint32_t* projection, size_t n_projection,
                 int keep_builtin, struct ArrowArrayStream* out);

int hg_compact_open(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                    struct ArrowArrayStream* out);

/* The resolved writer options of ONE column (WriteConfig's table-wide fields overridden by column_options[name], config.rs:54-133):
 * what parquet-rs writes for that column as build_write_props (storage.rs:258-298) configures it. */
typedef struct {
  uint8_t encoding;     /* 0 PLAIN, 5 DELTA_BINARY_PACKED (integer columns only): the chunk's encoding, or its fallback when a dictionary
                           is refused.  Any other value: HG_ERR_UNSUPPORTED */
  uint8_t dictionary;   /* 1: PLAIN dictionary page (first-appearance order, keys = physical bits) + RLE_DICTIONARY data page; a chunk
                           whose dictionary page would exceed 1 MiB (parquet-rs's dictionary_page_size_limit) falls back to `encoding` */
  uint8_t codec;        /* 0 UNCOMPRESSED, 1 SNAPPY, 6 ZSTD; the dictionary page is compressed with its chunk's codec */
  uint8_t bloom_filter; /* 1: one split-block bloom filter per chunk of this column (enable_bloom_filter, config.rs:100 / 113), hashed
                           from the non-null values' PLAIN bytes, written after its row group's chunks; 0: none.  Other values:
                           HG_ERR_UNSUPPORTED */
} hg_column_write_opts;

/* build_write_props (storage.rs:258-298) / WriteConfig (config.rs:120-133) as far as the GPU writer implements them:
 * PLAIN / DELTA_BINARY_PACKED / dictionary pages, RLE definition levels, optional bloom filters, chunk statistics on, one DataPage V1
 * per chunk (plus its dictionary page). */
typedef struct {
  uint32_t max_row_group_size;      /* 0 = 8192 (WriteConfig::default) */
  uint32_t compression;             /* Parquet codec id the WRITER applies: 0 UNCOMPRESSED, 1 SNAPPY (the default), 6 ZSTD (config.rs:78-94:
                                       Uncompressed / Snappy / Zstd; one frame per page, no level knob, like ZstdLevel::default()).
                                       Any other value: HG_ERR_UNSUPPORTED.  Zstd SSTs are read on the general pipeline */
  uint32_t enable_sorting_columns;  /* sorting_columns = primary keys, ascending, nulls first */
  uint32_t bloom_filter_bytes;      /* bitset size of every bloom filter: 0 = 1 MiB (parquet-rs's default ndv 1,000,000 at fpp 0.05);
                                       else a power of two in [32, 128 MiB], any other value: HG_ERR_INVALID */
  const hg_column_write_opts* columns;   /* NULL: every column PLAIN, no dictionary, no bloom filter, codec `compression` (the same bytes
                                            as an explicit all-PLAIN array); else schema->num_columns entries, __seq__ and __reserved__ included, and
                                            `compression` is ignored.  SSTs with DELTA or dictionary pages are read on the general pipeline */
} hg_write_props;

/* FileMeta (sst.rs:155-160) of the file just written.  num_rows / size are u32 in the reference: larger outputs are refused. */
typedef struct {
  uint64_t size;
  uint32_t num_rows, _pad;
  int64_t time_start, time_end;     /* union of the inputs' ranges (executor.rs:157-163) */
  uint64_t max_sequence;            /* max over the inputs */
} hg_file_meta;

/* Executor::do_compaction end to end on the GPU (compaction/executor.rs:155-222): merge + dedup of the input SSTs (builtin
 * columns kept) AND the Parquet encode of the result, written to `out_path` ("{root}/data/{id}.sst", sst.rs:202-204).
 * The Rust side keeps the manifest update (executor.rs:206-216). */
int hg_compact_to_sst(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* shard_preds,
                      size_t n_shard_preds, const hg_write_props* props, const char* out_path, hg_file_meta* out);
/* `shard_preds` (normally none) restricts the compaction to a primary-key range: the multi-GPU split of SURVEY 8(e) — GPU g
 * compacts `pk0 >= splitter[g-1] AND pk0 < splitter[g]` of ALL inputs (only the row groups overlapping its range are read:
 * SSTs are PK-sorted), the outputs concatenated in rank order are the globally sorted, deduplicated run.  A range on pk0
 * never cuts a primary-key run, so LastValue sees every version of a key on one GPU.
 *
 * hg_plan_pk_splitters: host only, deterministic — every rank computes the same `parts - 1` splitters (pk0 values in the
 * column's widened domain: i64 / u64 two's complement) from the row-group statistics of the inputs, balancing rows. */
int hg_plan_pk_splitters(const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, uint32_t parts, uint64_t* splitters);

/* ObjectBasedStorage::write_batch on the GPU (storage.rs:189-225): sort the batch by its primary keys (sort_batch, storage.rs:244-256:
 * ascending; equal keys keep their input order), append __seq__ = `sequence` and an all-null __reserved__ (fill_builtin_columns,
 * types.rs:219-239), encode with the writer above and write `out_path`.  `batch` is an Arrow C struct array holding the USER columns
 * (schema->num_columns - 2 children, primitive types matching schema->types); it stays owned by the caller.
 * NULL primary keys are refused (HG_ERR_UNSUPPORTED), like everywhere else on the GPU path. */
int hg_write_batch(hg_engine* e, const hg_schema_desc* schema, const struct ArrowArray* batch, uint64_t sequence, const hg_write_props* props,
                   const char* out_path, hg_file_meta* out);

int hg_scan_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                      const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg,
                      struct ArrowArrayStream* out);

/* Counter aggregates (Prometheus-style counters: rate() / increase()) per (series, bucket), on the deduplicated stream; an
 * overwritten older version of a sample never takes part.  `agg` is read as for hg_scan_aggregate, with these requirements:
 *   value_col >= 0, an integer or float column (Binary: HG_ERR_INVALID); ts_col >= 0, an integer column (HG_ERR_INVALID);
 *   the key is the sort prefix, so that a group is one series in time order: num_primary_keys >= 2, group_col == 0, ts_col == 1
 *   (else HG_ERR_UNSUPPORTED); mode HG_AGG_RUNS or HG_AGG_HASH, identical for this key (above: HG_ERR_INVALID); an Append-mode
 *   schema is HG_ERR_UNSUPPORTED.  Every check runs before any device work.
 * window_ms > 0 buckets exactly as hg_scan_aggregate (truncate_by); window_ms <= 0 makes one group per series.
 * The stream's columns, groups in key order:
 *   <group column name> (native), bucket (i64, only when window_ms > 0), count (u64: the group's rows, NULL values included),
 *   first_ts (i64), first_value (f64): the first row with a non-NULL value; last_ts (i64), last_value (f64): the last one,
 *   increase (f64), resets (u64).
 * first_* / last_* are NULL when the group has no non-NULL value; then increase = 0.0 and resets = 0.  Times are the time column
 * widened to i64.  Over the group's non-NULL values v1..vm in stream order, each converted to f64 (an integer counter above 2^53
 * is rounded first, so its differences are differences of rounded values):
 *   resets   = #{ i >= 2 : v_i < v_(i-1) }           (IEEE <: a NaN is never a reset)
 *   increase = 0.0, then for i = 2..m: increase += (v_i < v_(i-1)) ? v_i : v_i - v_(i-1), strictly in this order
 * (a drop is a counter restart from 0).  Bucket partials compose into longer ranges: over buckets b = 1..k of a series,
 *   increase = sum_b increase_b + sum_(b<k) (first_(b+1) < last_b ? first_(b+1) : first_(b+1) - last_b), and resets likewise
 *   (sum_b resets_b + the boundaries with first_(b+1) < last_b), where first / last are first_value / last_value.
 * Runs on the general pipeline (stats.path = 0).  Like every call, it ends the lifetime of the previous hg_scan_aggregate_device result. */
int hg_scan_counter_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                              const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg,
                              struct ArrowArrayStream* out);

/* Quantile aggregates (p50 / p90 / p99 of a gauge; PromQL quantile_over_time) per group and bucket, on the deduplicated stream; an
 * overwritten older version of a row never takes part.  `agg` is read as for hg_scan_aggregate: any non-Binary group_col, or -1 for one
 * global group; ts_col with window_ms > 0 for buckets (truncate_by); mode HG_AGG_RUNS or HG_AGG_HASH with the same groups in the same order.
 * value_col is required, an integer or float column.  `quantiles[0 .. n_quantiles)` are the q's, in any order, duplicates allowed.
 * Refused before any device work:  HG_ERR_INVALID: quantiles == NULL, n_quantiles 0 or above HG_MAX_QUANTILES, a q that is NaN or outside
 * [0, 1], value_col < 0, a Binary value / group / time column, a float time column with buckets, a bad mode;  HG_ERR_UNSUPPORTED: an
 * Append-mode schema.
 * The stream's columns:  <group column name> (native; absent when group_col = -1), bucket (i64, only when window_ms > 0), count (u64: the
 * group's rows, NULL values included), quantile_0 .. quantile_(n-1) (f64, in the caller's order).  Key, bucket and count equal
 * hg_scan_aggregate's for the same spec under HG_FLAG_NO_FUSED.
 * Definition (bit-exact).  Take the group's m non-NULL values and order them by the value domain's order (order_key: integers
 * numerically, floats in IEEE totalOrder, -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN); convert each selected value to f64 (an
 * integer above 2^53 is rounded; the conversion is monotone).  With v(0) <= ... <= v(m-1), for each q:
 *   rank = q * (m - 1),  lo = floor(rank),  hi = min(lo + 1, m - 1),  w = rank - lo,
 *   result = w == 0 ? v(lo) : v(lo) * (1 - w) + v(hi) * w,
 * every operation rounded to nearest f64 on its own (no fused multiply-add).  This is the interpolation of Prometheus's
 * quantile_over_time, and numpy's / pandas' "linear" method up to their rounding.  When m = 0 every quantile of the group is NULL.
 * Quantiles do not combine from partials: hg_agg_combine does not apply.  Runs on the general pipeline (stats.path = 0).  Like every
 * call, it ends the lifetime of the previous hg_scan_aggregate_device result. */
#define HG_MAX_QUANTILES 16u
int hg_scan_quantile_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                               const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg,
                               const double* quantiles, uint32_t n_quantiles, struct ArrowArrayStream* out);

int hg_scan_aggregate_device(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                             const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg,
                             hg_agg_device* out);

/* Aggregates by label group.  The data table holds series ids, not labels: the caller's index lookup finds the series a query selects
 * and the label group of each (e.g. the `job` value of `sum by (job)`), and passes them as a series -> group map.  Row r belongs to
 * group groups[i] when its agg->group_col value equals keys[i].  keys are in the column's widened domain (i64 / u64 two's complement, as
 * HG_OP_IN_SET's in_values), in any order; a key may repeat only with the same group.  groups are the caller's ordinals (e.g. an index
 * into the label-value combinations it found), any u32. */
typedef struct {
  const uint64_t* keys;
  const uint32_t* groups;
  uint32_t count, _pad;        /* 0 .. HG_MAX_IN_SET */
} hg_group_map;

/* The calls by map.  Every one of them reads `agg` as hg_scan_aggregate does, with group_col naming the key column of the map:
 * - Rows: as if `group_col IN_SET map.keys` were one more predicate after the caller's, with HG_OP_IN_SET's rules: it filters before
 *   the merge and dedup, a NULL key never matches, an empty map matches no row.  Row groups are pruned by that set exactly as for
 *   HG_OP_IN_SET, and transient loads ship only their surviving row groups.
 * - Groups: every row of the deduplicated stream that survives belongs to group map(key).
 * - Count / sum / min / max (hg_scan_aggregate_by_map): hg_scan_aggregate in HASH mode over a u32 group column whose value on every row
 *   is map(key): every group's rows are added in stream order, groups come out sorted by (group ordinal, bucket).
 * - ts_col / window_ms bucket exactly as hg_scan_aggregate (truncate_by); mode HG_AGG_RUNS and HG_AGG_HASH are both accepted and give
 *   the same result.
 * - Quantiles (hg_scan_quantile_aggregate_by_map): the same groups, each with hg_scan_quantile_aggregate's bit-exact definition.
 * - The stream's columns: group (u32), bucket (i64, only when window_ms > 0), count (u64), then sum / min / max (f64, when value_col >= 0)
 *   or quantile_0 .. quantile_(n-1), named and defined as by hg_scan_aggregate / hg_scan_quantile_aggregate.
 * - hg_scan_aggregate_by_map_device fills hg_agg_device with d_gkey = the u32 ordinals: hg_agg_export_packed zero-extends them and
 *   hg_agg_combine (GATHER and REDUCE) works unchanged, so label groups that cross ranks combine with HG_COMBINE_REDUCE.
 * - Refused before any device work:  HG_ERR_INVALID: map == NULL; keys or groups NULL with count > 0; count above HG_MAX_IN_SET; a key
 *   mapped to two different groups; group_col < 0; a Binary key / value / time column; a float time column with buckets; a bad mode;
 *   the quantile call's checks of hg_scan_quantile_aggregate.  HG_ERR_UNSUPPORTED: a float key column (as for HG_OP_IN_SET); an
 *   Append-mode schema; more than 7 caller predicates (with the map's, more than 8).
 * - Stats: path = 0 (the general pipeline, whole pages), groups_out = the groups; rows_filtered counts the map's membership test too and
 *   bytes_h2d the map's upload (its keys, as the set of the IN_SET predicate, and its groups).
 * Like every call, each ends the lifetime of the previous hg_scan_aggregate_device result. */
int hg_scan_aggregate_by_map(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                             const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg, const hg_group_map* map,
                             struct ArrowArrayStream* out);
int hg_scan_aggregate_by_map_device(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                                    const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg, const hg_group_map* map,
                                    hg_agg_device* out);
int hg_scan_quantile_aggregate_by_map(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                                      const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg, const hg_group_map* map,
                                      const double* quantiles, uint32_t n_quantiles, struct ArrowArrayStream* out);

/* Packs the last hg_scan_aggregate_device result into a caller-owned device buffer of 6 x cap int64 words
 * (rows: group key, bucket, count, sum bits, min bits, max bits; columns >= num_groups are zero) on the engine's stream:
 * the block one NCCL all-gather combines across GPUs.  HG_ERR_INVALID if cap < num_groups. */
int hg_agg_export_packed(hg_engine* e, void* d_dst, uint64_t cap);

int hg_last_stats(hg_engine* e, hg_scan_stats* out);

/* ---- multi-GPU combine of the per-GPU partial aggregates (SURVEY 8e): one engine per GPU / process, NCCL over NVLink.
 * The aggregation stage and its combine are absent in the reference (metric_engine/src/metric/mod.rs:37-49 is todo!());
 * SSTs shard by file (one partition per SST, read.rs:442-450), so every rank scans its own files and ONE collective
 * combines the partials.  The host ships the NCCL id between ranks over its own channel. */
#define HG_COMM_ID_BYTES 128
typedef enum {
  HG_COMBINE_GATHER = 0,  /* partials are disjoint (keys contain the series id): all-gather of the packed blocks */
  HG_COMBINE_REDUCE = 1   /* keys cross ranks (per-(tag, bucket)): all-gather + per-group combine on every rank: counts summed,
                             min / max taken, f64 sums added in RANK order (deterministic) */
} hg_combine_mode;
typedef struct {
  uint64_t capacity;          /* columns per rank block */
  uint32_t world, _pad;
  const int64_t* d_blocks;    /* device, [world][6][capacity] int64: rows key, bucket, count, sum / min / max bits; count == 0 pads */
  uint64_t num_groups;        /* REDUCE: groups of the combined table */
  uint64_t reduced_capacity;
  const int64_t* d_reduced;   /* REDUCE: device, [6][reduced_capacity], sorted by (key, bucket); identical on every rank */
} hg_agg_combined;
int hg_comm_unique_id(uint8_t* id /* HG_COMM_ID_BYTES */);
int hg_comm_init(hg_engine* e, const uint8_t* id, int rank, int world);
int hg_comm_destroy(hg_engine* e);
/* Collective over all ranks of the communicator: combines the results of their last hg_scan_aggregate_device calls.  The pack
 * kernel runs on the engine stream behind the scan, the collective on the engine's combine stream (the next scan overlaps it);
 * GATHER results are valid after hg_comm_sync.  capacity_hint = 0: the ranks first agree on the block width (one extra small
 * collective + host sync); > 0: every rank passes the same value and promises num_groups <= capacity_hint. */
int hg_agg_combine(hg_engine* e, uint32_t mode, uint64_t capacity_hint, hg_agg_combined* out);
int hg_comm_sync(hg_engine* e);

/* ---- host-only inspection of an SST (no engine, no GPU): what the planner reads from the footer and the page headers.
 * In the reference this is parquet-rs's metadata reader behind ParquetExec (read.rs:66-93, 442-465); the CPU test-suite
 * checks it against pyarrow's reading of the same bytes. */
typedef struct {
  uint64_t num_rows;
  uint32_t num_row_groups, num_columns;
  uint64_t num_data_pages;
  uint64_t sum_page_values;          /* sum of num_values over all data pages */
  uint64_t sum_uncompressed_bytes;   /* sum of uncompressed page payload sizes (page headers excluded) */
  uint64_t sum_compressed_bytes;     /* the same, as stored */
  uint32_t codec_mask;               /* bit c set: some column chunk uses Parquet codec id c (0 uncompressed, 1 Snappy, 6 Zstd) */
  uint32_t max_pages_per_chunk;
} hg_parquet_summary;

typedef struct {
  uint64_t num_rows;                 /* rows of the row group */
  uint64_t num_values;               /* values of the column chunk (nulls included) */
  int64_t data_page_offset, total_compressed_size;
  int64_t null_count;                /* -1: not recorded */
  uint8_t min[8], max[8];            /* PLAIN-encoded statistics (little endian), valid if has_min_max */
  uint32_t has_min_max, physical_type, codec, num_pages;
  uint64_t first_page_payload_offset;
  uint32_t first_page_num_values, first_page_type;   /* 0 = DataPage V1, 3 = DataPage V2 */
} hg_parquet_chunk;

/* The planner's row-group pruning for ONE SST, host only: keep[g] = 1 iff row group g can hold a row matching the
 * conjunction (DataFusion's PruningPredicate as pinned by the plan text at read.rs:613: CASE WHEN null_count = row_count
 * THEN false ELSE <min/max rewrite> END; then its bloom filters for `=` / `IN` predicates, as bloom_filter_on_read does).  Also runs the schema / predicate / file validation every scan call runs.
 * HG_ERR_INVALID if cap < number of row groups. */
int hg_plan_row_groups(const hg_schema_desc* schema, const uint8_t* data, uint64_t size, const hg_predicate* preds, size_t n_preds,
                       uint8_t* keep, uint32_t cap, uint32_t* num_row_groups);

int hg_parquet_inspect(const uint8_t* data, uint64_t size, hg_parquet_summary* out);
int hg_parquet_chunk_info(const uint8_t* data, uint64_t size, uint32_t row_group, uint32_t column, hg_parquet_chunk* out);

/* The bloom filter of one column chunk (ColumnMetaData.bloom_filter_offset / _length) as the planner sees it.  usable = 0: the chunk
 * has none, or its header, size or range is malformed, or its algorithm / hash / compression is not SBBF / XXHASH / UNCOMPRESSED (such
 * a filter is ignored: it never prunes).  Binary chunks keep no filter. */
typedef struct {
  int64_t offset;                    /* bloom_filter_offset: file offset of the BloomFilterHeader; -1 if absent */
  int32_t length;                    /* bloom_filter_length (header + bitset); -1 if absent */
  uint32_t num_bytes;                /* BloomFilterHeader.numBytes when usable */
  uint64_t bitset_offset;            /* file offset of the bitset when usable */
  uint32_t usable, _pad;
} hg_parquet_bloom;
int hg_parquet_bloom_info(const uint8_t* data, uint64_t size, uint32_t row_group, uint32_t column, hg_parquet_bloom* out);
/* Probes that filter with the PLAIN physical bytes of one value (len 4 or 8): *maybe = 0 only if the value is certainly absent;
 * a chunk without a usable filter gives *maybe = 1. */
int hg_parquet_bloom_probe(const uint8_t* data, uint64_t size, uint32_t row_group, uint32_t column, const void* value, uint32_t len,
                           int* maybe);

#ifdef __cplusplus
}
#endif
#endif /* HORAE_GPU_H */
