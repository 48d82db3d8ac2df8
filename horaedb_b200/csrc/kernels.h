// kernels.h — host-callable launch wrappers of the sm_90a kernels (kernels.cu, fused_scan.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "device_types.h"

namespace horae {

// Streaming multiprocessors of the target GPU (H100 SXM).  Grid-stride and ticket-driven kernels size their grids as a
// multiple of it; results never depend on the grid size.  The CPU emulation of the test suite (tests/emu) runs every thread
// as a coroutine: 4 "SMs" still exercise tickets, look-backs and last-block patterns without repeating them on empty work.
#ifdef HORAE_EMULATED_BUILD
constexpr int kNumSMs = 4;
#else
constexpr int kNumSMs = 132;
#endif

// blocks of a grid-stride kernel over n items: one per `per_block` items, at least 1, at most max_blocks
inline int grid_for(uint64_t n, int per_block = 256, int max_blocks = kNumSMs * 16) {
  uint64_t b = (n + per_block - 1) / per_block;
  if (b < 1) b = 1;
  return int(b > uint64_t(max_blocks) ? max_blocks : b);
}

struct Launch {
  cudaStream_t stream;
  uint32_t* counter;  // host-side count of kernels launched (reported as hg_scan_stats.kernel_launches)
  void tick() const { if (counter) ++*counter; }
};

namespace k {

// S2: page decompression + decode --------------------------------------------------------------------------------
// Snappy pages of the selected chunks -> scratch (snappy.cu, decoder in snappy_core.h); `ticket` is a zeroed device counter
void snappy_chunks(const Launch& L, const SstDev* ssts, const RgSel* sel, uint32_t nsel, const ColSel* cols, int ncolsel,
                   uint8_t* scratch, unsigned int* ticket, int* err);
// The same decompressor driven by a job descriptor (fused Snappy path: row-group list and its length live on the device,
// every (row group, column) gets a fixed-size scratch region addressed by RgSel::scratch_off + region * fixed_stride).
constexpr int kSnappyMaxCols = 32;
struct SnappyJob {
  const SstDev* ssts;
  const RgSel* sel;
  const uint32_t* d_nsel;     // device-side count of row groups, or nullptr: use nsel
  const uint32_t* lpt;        // optional: row-group indices in the order the tickets hand them out (longest pages first)
  uint32_t nsel;
  int ncols;                  // columns to decompress per row group
  uint32_t col[kSnappyMaxCols];        // schema column of entry i
  uint32_t region[kSnappyMaxCols];     // fixed_stride != 0: scratch region index of entry i inside the row group's block
  uint8_t order[kSnappyMaxCols];       // processing order of the entries (heaviest column first)
  uint8_t skip_stored[kSnappyMaxCols]; // entry i: leave stored (literal-only) pages alone, the consumer reads them in place
  uint8_t partial[kSnappyMaxCols];     // entry i: only rows [0, RgSel::out_row) of the (single) page are needed: stop decompressing there
  const ColSel* cols;         // general pipeline: column ids + variable scratch offsets come from the ColSel table
  int col_from_cols;
  uint64_t fixed_stride;      // bytes per scratch region, 0 = general pipeline layout
  uint8_t* scratch;
  unsigned int* ticket;       // zeroed device counter
  int* err;
};
void snappy_pages(const Launch& L, const SnappyJob& job, uint32_t max_chunks);
// Zstandard pages of the selected chunks -> scratch (zstd.cu); `ticket` is a zeroed device counter
void zstd_chunks(const Launch& L, const SstDev* ssts, const RgSel* sel, uint32_t nsel, const ColSel* cols, int ncolsel, uint8_t* scratch,
                 unsigned int* ticket, int* err);
// raw Snappy streams by pointer: dst must be 16-byte aligned with uncomp_size + 48 bytes of room; ticket = zeroed device counter
struct RawPage { const uint8_t* src; uint8_t* dst; uint32_t comp_size, uncomp_size; };
void snappy_raw_pages(const Launch& L, const RawPage* d_pages, uint32_t n, unsigned int* ticket, int* err);
// dba / dba_base: the call's DELTA_BYTE_ARRAY page descriptors, and per (row group, column) block the index of its first one (both
// nullptr when the selected chunks have no such page)
void decode_chunks(const Launch& L, const SstDev* ssts, const RgSel* sel, uint32_t nsel, const ColSel* cols,
                   int ncolsel, uint8_t* scratch, DbaPage* dba, const uint32_t* dba_base, int* err);
// values of the DELTA_BYTE_ARRAY pages sized by decode_chunks (out_off set by the host), written at out + out_off; rows point there
void dba_materialise(const Launch& L, const DbaPage* pages, uint32_t npages, const ColSel* cols, uint8_t* out);

// S3: predicate -> alive bytes -----------------------------------------------------------------------------------
void eval_predicates(const Launch& L, const PredSet& preds, uint32_t n, uint8_t* alive);
// the Binary predicates of the conjunction: and_alive = AND into the bytes eval_predicates wrote, else write them
void eval_binary_predicates(const Launch& L, const BinPredSet& preds, uint32_t n, bool and_alive, uint8_t* alive);
// the OP_IN_SET predicates of the conjunction (kernels.cu: eval_in_set_kernel), one tile of kInSetTile rows per block step; a tile's slice
// of a set is searched in shared memory when it has at most kInSetSmemKeys keys, through that many splitters otherwise
constexpr uint32_t kInSetTile = 2048;
constexpr uint32_t kInSetSmemKeys = 4096;
void eval_in_set(const Launch& L, const InSetPreds& preds, uint32_t n, bool and_alive, uint8_t* alive);
// A2 by map (kernels.cu: group_map_kernel, the same tiled search): out[rows[t]] = groups[i] for every deduplicated row t < *d_r whose key
// column's order key is keys[i] (sorted, unique).  Those rows all passed `col IN_SET keys`: a row without its key in the set is an
// internal error, reported as *err = kErrGroupMapMiss with its group left unwritten.
constexpr int kErrGroupMapMiss = 150;
void group_map(const Launch& L, ColView col, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, const uint64_t* keys, const uint32_t* groups,
               uint32_t n_keys, uint32_t* out, int* err);

// stream compaction: indices of non-zero flag bytes, in order.  tmp must hold (n/2048+2) uint32.  *d_total = count.
void compact_flags(const Launch& L, const uint8_t* flags, uint32_t n, uint32_t* tmp, uint32_t* out_idx,
                   uint32_t* d_total);
size_t compact_tmp_elems(uint32_t n);

// S4: k-way merge on (pk..., __seq__) ----------------------------------------------------------------------------
// run_start[f] = first survivor index of file f (k+1 entries, device); derived from decoded-row file bases.
void survivor_run_starts(const Launch& L, const uint32_t* surv, const uint32_t* d_m, const uint32_t* file_base,
                         int k, uint32_t* run_start);
void build_records(const Launch& L, const PkSet& pk, ColView seq, const uint32_t* surv, const uint32_t* d_m,
                   uint32_t cap, SortRec* rec);
// one pairwise pass = partition kernel (merge-path split per 1024-record tile) + merge kernel; splits holds
// merge_split_elems(cap) uint32
void merge_pass(const Launch& L, const SortRec* src, SortRec* dst, const uint32_t* run_start, int k, int level,
                const uint32_t* d_m, uint32_t cap, uint32_t* splits);
size_t merge_split_elems(uint32_t cap);
// Single-pass k-way merge over packed 64-bit keys (kway_merge.cu).  KeyPack = how (pk..., __seq__, stream) packs into
// 52 bits: every field rebased to its minimum over the selected row groups (chunk statistics), stream index lowest.
constexpr int kMaxMergeRuns = 128;
struct KeyPack {
  uint64_t mn[MAX_PK], span[MAX_PK];
  uint32_t shift[MAX_PK];
  uint64_t seq_min, seq_span;      // in the (value + 1, NULL = 0) domain of the sort records
  uint32_t seq_shift, pk_shift;    // pk_shift = bits below the primary-key part (seq + stream)
};
// tmp must hold kway_tmp_bytes(cap, k, &ranges) bytes; order[j] = row id of the j-th merged record, keep[j] = 1 iff it is
// the last of its primary-key run (== records_to_rows + dedup_flags_recs after the pairwise passes).
size_t kway_tmp_bytes(uint32_t cap, int k, uint32_t* ranges);
void kway_merge(const Launch& L, const PkSet& pk, ColView seq, const uint32_t* surv, const uint32_t* d_m, uint32_t cap, const uint32_t* run_start,
                int k, const KeyPack& kp, void* tmp, unsigned int* ticket, uint32_t* order, uint8_t* keep, int* err);
void records_to_rows(const Launch& L, const SortRec* rec, const uint32_t* d_m, uint32_t cap, uint32_t* order);

// S5/S6: PK-run boundaries, LastValue = keep the last row of each run ---------------------------------------------
// order == nullptr means identity.  keep[j] = 1 iff row order[j] is the last of its PK run in the merged stream.
void dedup_flags_cols(const Launch& L, const PkSet& pk, const uint32_t* order, const uint32_t* d_m, uint32_t cap,
                      uint8_t* keep);
void dedup_flags_recs(const Launch& L, const SortRec* rec, const uint32_t* d_m, uint32_t cap, uint8_t* keep);
// out_rows[r] = order[out_pos[r]]
void gather_rows(const Launch& L, const uint32_t* order, const uint32_t* out_pos, const uint32_t* d_r, uint32_t cap,
                 uint32_t* out_rows);
// bound[c] = #outputs whose merged position < chunk_end[c] - 1   (batch boundaries of MergeStream, read.rs:289-343)
void batch_bounds(const Launch& L, const uint32_t* out_pos, const uint32_t* d_r, const uint32_t* chunk_end,
                  uint32_t nchunks, uint32_t* bound);
// chunk_end for the single-SST pass-through: #survivors before each reader-batch boundary row
void chunk_ends_from_rows(const Launch& L, const uint32_t* surv, const uint32_t* d_m, const uint32_t* piece_end_row,
                          uint32_t npieces, uint32_t* chunk_end);

// output materialisation ------------------------------------------------------------------------------------------
void gather_column(const Launch& L, ColView src, const uint32_t* rows, const uint32_t* d_r, uint32_t cap,
                   void* dst_vals, uint8_t* dst_valid);
void pack_validity(const Launch& L, const uint8_t* valid_bytes, uint32_t n, uint8_t* bitmap,
                   unsigned long long* null_count);

// A1/A2: time-bucket aggregation over the post-dedup stream -------------------------------------------------------
void group_flags(const Launch& L, const AggSpecDev& spec, const uint32_t* rows, const uint32_t* d_r, uint32_t cap,
                 uint8_t* head);
void reduce_groups(const Launch& L, const AggSpecDev& spec, const uint32_t* rows, const uint32_t* d_r,
                   const uint32_t* seg_start, const uint32_t* d_g, uint32_t cap, AggOut out);
// counter partials per group (the same inputs as reduce_groups; spec.ts must be set even without buckets: first_ts / last_ts)
void reduce_counter_groups(const Launch& L, const AggSpecDev& spec, const uint32_t* rows, const uint32_t* d_r,
                           const uint32_t* seg_start, const uint32_t* d_g, uint32_t cap, CounterOut out);

// kernels.cu (quantile_*): exact quantiles per group (hg_scan_quantile_aggregate).  quantile_prepare takes the groups of group_rows and leaves, per
// group, its slice of the non-NULL values' order keys and its tier; the host reads counters[0 .. kQuantileCounters) and quantile_select
// launches only the tiers that have groups.  A group of m non-NULL values is small up to kQuantileSmallMax (one warp), medium up to
// kQuantileMediumMax (one block) and large above (radix select in 8 passes; a group above kQuantileChunk spans several blocks a pass).
constexpr uint32_t kQuantileMax = 16;                 // HG_MAX_QUANTILES
constexpr uint32_t kQuantileSmallMax = 32;
constexpr uint32_t kQuantileMediumMax = 4096;
constexpr uint32_t kQuantileChunk = 16384;
struct QuantileSpec { double q[kQuantileMax]; uint32_t n; };
struct QuantileGroup { uint32_t g, start, m; };       // group g's keys are keys[start, start + m)
struct QuantileLarge {                                // a large group's selection state: the sorted distinct ranks it needs
  uint32_t g, start, m, nr;
  uint32_t chunk, _pad;                                       // the group's first chunk of kQuantileChunk keys among all large groups
  uint32_t rank[2 * kQuantileMax], left[2 * kQuantileMax];   // left: the rank within the keys that match prefix
  uint64_t prefix[2 * kQuantileMax];                          // the digits resolved so far
};
// QC_LARGE_CHUNKS / QC_LARGE are the low / high word of one 64-bit counter (8-byte aligned)
enum : uint32_t { QC_VALUES = 0, QC_SMALL, QC_MEDIUM, QC_MEDIUM_MAX, QC_LARGE_CHUNKS = 6, QC_LARGE = 7, kQuantileCounters = 8 };
struct QuantileBufs {
  uint8_t* flags;          // [cap]
  uint32_t* compact_tmp;   // [compact_tmp_elems(cap)]
  uint32_t* idx;           // [cap]: agg rows with a non-NULL value, in order
  uint64_t* keys;          // [cap]: their order keys
  QuantileGroup* list;     // [G]: small groups from the front, medium groups from the back
  QuantileLarge* large;    // [quantile_large_cap(cap)]
  uint32_t* hist;          // [quantile_hist_elems(large groups)], zeroed
  uint32_t* counters;      // [kQuantileCounters], zeroed
  double* out;             // [n][G]: quantile j of group g at out[j * G + g] (0.0 for a group without values)
  uint8_t* valid;          // [G]: the group has a non-NULL value
};
size_t quantile_large_cap(uint32_t cap);
size_t quantile_hist_elems(uint32_t n_large);
void quantile_prepare(const Launch& L, ColView value, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, const uint32_t* seg,
                      const uint32_t* d_g, uint32_t G, const QuantileSpec& qs, const QuantileBufs& b);
void quantile_select(const Launch& L, const QuantileSpec& qs, uint32_t type, uint32_t G, const uint32_t host_counters[kQuantileCounters],
                     const QuantileBufs& b);

// radix_agg.cu: stable LSD radix sort of (key, row) pairs by key bits [0, bits); count on the device.  Returns 0 if the
// result is in (keys, vals), 1 if in (keys_tmp, vals_tmp).  counts: radix_tmp_elems(cap) uint32.
size_t radix_tmp_elems(uint32_t cap);
int radix_sort_pairs(const Launch& L, uint64_t* keys, uint32_t* vals, uint64_t* keys_tmp, uint32_t* vals_tmp, const uint32_t* d_n, uint32_t cap,
                     int bits, uint32_t* counts);
// order-preserving sort keys of the rows `rows[0..*d_r)`: gk = group value, bk = bucket start (either may be null); vals = rows
void group_sort_keys(const Launch& L, const AggSpecDev& spec, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, uint64_t* gk, uint64_t* bk,
                     uint32_t* vals);
// Binary (variable-width) columns: export helpers.  gather_lens: byte length per output row (0 beyond *d_n / for NULL);
// exclusive_scan_u32: single-block in-place exclusive scan of n words (*d_total = sum, when d_total is given); copy_var: bytes of row rows[i] -> dst + offs[i];
// first_rows / run_offsets: Append mode (BytesMergeOperator): the runs' first rows, the offsets of the concatenated values.
void gather_lens(const Launch& L, ColView col, const uint32_t* rows, const uint32_t* d_n, uint32_t cap, uint32_t* out);
void copy_var(const Launch& L, ColView col, const uint32_t* rows, const uint32_t* d_n, uint32_t cap, const uint32_t* offs, uint8_t* dst);
void first_rows(const Launch& L, const uint32_t* order, const uint32_t* out_pos, const uint32_t* d_r, uint32_t cap, uint32_t* out);
void run_offsets(const Launch& L, const uint32_t* cum, const uint32_t* out_pos, const uint32_t* d_r, const uint32_t* d_m, uint32_t cap, uint32_t* out);
// validity of a run's concatenated value (operator.rs:80-92: a run whose bytes are empty returns its column UNCHANGED — one row keeps
// its own validity; several rows cannot be assembled into the one-row batch, which the reference reports as an error: *err = 130)
void append_validity(const Launch& L, ColView col, const uint32_t* order, const uint32_t* out_pos, const uint32_t* d_r, const uint32_t* run_offs,
                     uint32_t cap, uint8_t* valid, int* err);
void exclusive_scan_u32(const Launch& L, uint32_t* data, uint32_t n, uint32_t* d_total);
// write path helpers (radix_agg.cu)
void column_sort_keys(const Launch& L, ColView col, const uint32_t* perm, uint32_t n, uint64_t* keys);
void iota_u32(const Launch& L, uint32_t* p, uint32_t n);
void fill_u64(const Launch& L, uint64_t* p, uint64_t v, uint32_t n);
void unpack_bitmap(const Launch& L, const uint8_t* bitmap, uint64_t offset, uint32_t n, uint8_t* out);
void fill_u32(const Launch& L, uint32_t* p, uint32_t v, uint32_t n);
// dst[6][cap] int64: key, bucket, count, sum/min/max bit patterns; zero beyond g
void pack_agg(const Launch& L, AggOut in, uint32_t gwidth, uint64_t g, uint64_t cap, long long* dst);
// chunk_end[c] = min((c+1)*batch, *d_m): SortPreservingMergeExec re-batches its output at batch_size rows
void uniform_chunk_ends(const Launch& L, const uint32_t* d_m, uint32_t batch, uint32_t nchunks, uint32_t* chunk_end);
// flags[i] = 0 for i in [*d_n, cap)
void clear_tail(const Launch& L, uint8_t* flags, const uint32_t* d_n, uint32_t cap);

}  // namespace k
}  // namespace horae
