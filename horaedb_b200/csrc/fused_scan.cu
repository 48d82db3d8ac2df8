// fused_scan.cu — single-pass scan for the common metric-engine case: PK-disjoint (or single) SSTs whose needed column
// chunks are one uncompressed PLAIN page each.  One kernel reads the page payloads straight out of the resident SST
// bytes and does S2 (def-level skip + PLAIN decode), S3 (predicate), S5/S6 (PK-run dedup, last row wins) and A1/A2
// (group by pk0 [, time bucket of pk1]: count / sequential f64 sum / min / max) with no intermediate column ever
// written to HBM: algorithmic traffic = the bytes of the columns the query touches (SURVEY §8d: 24-28 B/row).
//
// Work decomposition: every selected row group is split into `split` (1..8) sub-ranges whose boundaries
// item_bounds_kernel moves to the next key-run start, so the work items are disjoint, cover the stream, and no group
// spans two of them.  One warp owns one item (taken from an atomic ticket, so all SMs x resident warps stay busy until the
// stream is exhausted) and sums its groups in strict stream order (bit-exact with the oracle) without any cross-warp
// communication.  Group records are appended unordered, tagged (item, local index), and a tiny scatter pass puts them
// in stream order.
//
// Late materialisation (GATED kernels): the narrowest predicate column is swept first, 512 rows per warp step; the other
// columns are read only for the 64-row blocks that hold a passing row, the value column only for survivors.  The
// reference filters before it merges and dedups (read.rs:459-480), so rows that fail the predicate take part in
// nothing downstream.
#include "fused_scan.h"

#include "block_scan.h"

#include <algorithm>
#include <cstddef>
#include <cstdlib>

namespace horae {
namespace fused {

namespace {

constexpr int MAXC = 8;
constexpr int kWarpsPerCta = 8;

struct alignas(16) FRec {
  uint32_t item, local;
  uint64_t gkey;
  int64_t bucket;
  uint64_t count;
  double sum, mn, mx;
  uint64_t _pad;
};

// In-place addressing of a stored (literal-only) Snappy page: rows [0, n0) start at the slot base, rows [n0, ..) at base1.
struct VSeg { const uint8_t* base1; uint32_t n0, _pad; };

enum : uint32_t { K_RAW64 = 0, K_U32 = 1, K_I32 = 2, K_F32 = 3 };   // how a PLAIN slot widens to 64 bits
inline uint32_t kind_of(uint32_t t) {
  return (t == T_U64 || t == T_I64 || t == T_F64) ? K_RAW64 : (t == T_F32 ? K_F32 : ((t == T_I8 || t == T_I16 || t == T_I32) ? K_I32 : K_U32));
}
// the order keys (widened value ^ sign bit) of i32's minimum and maximum: a signed 4-byte column's keys lie in between
constexpr uint64_t kI32KeyLo = (1ull << 63) - (1ull << 31), kI32KeyHi = (1ull << 63) + (1ull << 31) - 1;

struct FParams {
  const SstDev* ssts;
  const RgSel* sel;             // selected row groups in stream order, built on the device by select_rgs_kernel
  const uint32_t* d_nsel;       // their count
  const uint8_t* const* bases;  // [selected row group][MAXC]: start of the PLAIN values of every slot (slot_bases_kernel)
  uint32_t split;               // sub-ranges (work items) per row group
  uint32_t pcol[MAX_PREDS], pcls[MAX_PREDS];   // schema column / comparison class of every predicate (statistics pruning)
  uint32_t pbloom[MAX_PREDS];   // 1: an `=` predicate whose literal the column can represent: probe the chunk's bloom filter with phash
  uint64_t phash[MAX_PREDS];
  int nslots;
  uint32_t col[MAXC], kind[MAXC], cls[MAXC];
  int npk;                      // slots [0, npk) are the primary key columns in order
  int has_group, has_ts, value_slot, global_mode;
  // hot columns (position 0 = pk0, 1 = pk1, then predicate columns): loaded for every row.  The conjunction of all
  // predicates on one column is pre-compiled into ONE interval test in an order-preserving unsigned domain:
  //   key = value ^ flip ;  pass  <=>  key - lo <= span     (32-bit arithmetic for 4-byte columns)
  int hot_slot[kHot];
  uint64_t hot_flip[kHot], hot_lo[kHot], hot_span[kHot];
  int hot_haspred[kHot];
  // the same predicates in generic form, for the cold dedup look-ahead
  int npred;
  int pslot[MAX_PREDS];
  uint32_t pop[MAX_PREDS];
  uint64_t plit[MAX_PREDS];
  int64_t window_ms;
  // Snappy SSTs: pages are decompressed into fixed-size scratch regions first (snappy.cu); region r of selected row
  // group si starts at scratch + sel[si].scratch_off + r * scratch_stride
  const uint8_t* scratch;
  uint64_t scratch_stride;
  int region[MAXC];             // scratch region of slot s, -1 = the slot is never decompressed
  int value_stored;             // the value slot's Snappy pages are literal-only: read in place, in two segments (vseg)
  // gate bits (gate-first calls): the row-group gate (k::snappy_gate_pages for a 4-byte gate column, else gate_rg_kernel) writes one bit
  // per row of the gate column at scratch + sel[si].scratch_off + bits_off, and the gated kernel tests the gate column with them
  int gate_bits;
  int gate_slot;                // >= 0: that slot is a 4-byte gate column whose values are never decompressed (its bits stand for it)
  uint64_t bits_off;
  VSeg* vseg;                   // [selected row group]
  FRec* rec;
  uint32_t rec_cap;
  uint32_t* item_cnt;
  unsigned int* work;           // [0] item ticket, [1] record slots
  unsigned long long* counters; // [0] rows passing the predicate, [1] rows kept after dedup, [2] rows of selected row groups,
                                // [3] rows of blocks whose non-gate columns were loaded
  int* err;
};

// 8 bytes at ANY byte alignment, branch-free (two aligned 8-byte loads + funnel shift), so that the compiler can issue
// every load of a block back to back.  Buffers are padded: reading one aligned word past the value is always legal.
__device__ __forceinline__ uint64_t ld_bytes8(const uint8_t* p) {
  uintptr_t a = reinterpret_cast<uintptr_t>(p);
  uint32_t sh = uint32_t(a & 7) * 8;
  const uint64_t* q = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
  uint64_t lo = __ldg(q), hi = __ldg(q + 1);
  return (lo >> sh) | ((hi << 1) << (63 - sh));
}
__device__ __forceinline__ uint32_t ld32u(const uint8_t* p) { return uint32_t(ld_bytes8(p)); }

// widen the raw little-endian bytes of a PLAIN value: signed -> i64 bits, unsigned -> u64, floats -> f64 bits
__device__ __forceinline__ uint64_t widen_kind(uint64_t raw, uint32_t kind) {
  uint32_t r = uint32_t(raw);
  uint64_t v = raw;
  v = kind == K_U32 ? uint64_t(r) : v;
  v = kind == K_I32 ? uint64_t(int64_t(int32_t(r))) : v;
  v = kind == K_F32 ? uint64_t(__double_as_longlong(double(__uint_as_float(r)))) : v;
  return v;
}
__device__ __forceinline__ uint64_t load_kind(const uint8_t* base, uint32_t kind, uint32_t row) {
  return widen_kind(ld_bytes8(base + size_t(row) * (kind == K_RAW64 ? 8u : 4u)), kind);
}

// Start of the PLAIN values of column slot `s` in selected row group `si`: a pointer chase through the resident tables
// (row group -> file -> chunk -> page -> def-level length), done once per (row group, slot) by slot_bases_kernel.
// literal element at p: header length and literal length (the caller knows it is a literal: stored pages only)
__device__ __forceinline__ uint32_t literal_header(const uint8_t* p, uint32_t* len) {
  const uint32_t t = __ldg(p);
  uint32_t l = t >> 2, hdr = 1;
  if (l >= 60) {
    const uint32_t nb = l - 59;
    l = 0;
    for (uint32_t i = 0; i < nb; i++) l |= uint32_t(__ldg(p + 1 + i)) << (8 * i);
    hdr = 1 + nb;
  }
  *len = l + 1;
  return hdr;
}

__device__ __forceinline__ const uint8_t* slot_base_chase(const FParams& P, uint32_t si, int s) {
  RgSel rs = P.sel[si];
  SstDev sst = P.ssts[rs.sst];
  ChunkDev cd = sst.chunks[size_t(rs.rg) * sst.ncols + P.col[s]];
  PageDev pg = sst.pages[cd.first_page];
  const uint8_t* body = sst.bytes + pg.payload_off;
  const bool is_value = P.value_stored && s == P.value_slot;
  if (cd.codec == 1) {
    if (is_value && cd.stored) {
      // stored page, read in place: [varint ulen][literal 0: level prefix + values][literal 1: values] (classify_stored)
      const uint8_t* p = body;
      while (__ldg(p) & 0x80) p++;
      p++;
      uint32_t len0 = 0, len1 = 0;
      const uint32_t h0 = literal_header(p, &len0);
      const uint8_t* lit0 = p + h0;
      const uint32_t prefix = cd.optional ? 4 + ld32u(lit0) : 0;
      const uint32_t w = P.kind[s] == K_RAW64 ? 8u : 4u;
      VSeg v;
      v.n0 = (len0 - prefix) / w;
      v._pad = 0;
      v.base1 = lit0 + prefix;
      if (lit0 + len0 < body + pg.comp_size) v.base1 = lit0 + len0 + literal_header(lit0 + len0, &len1);
      P.vseg[si] = v;
      return lit0 + prefix;
    }
    body = P.scratch + rs.scratch_off + uint64_t(P.region[s]) * P.scratch_stride;
  }
  if (cd.optional && s != P.gate_slot) {         // [u32 len][RLE def levels] — all-valid pages only (planner)
    uint32_t lv = ld32u(body);
    // the length comes out of the decompressed page: a damaged page — or one whose decompression stopped early (compressed prefix that
    // ran out: the call is repeated) — must not turn into a pointer outside the page
    if (lv > pg.uncomp_size) { lv = 0; atomicExch(P.err, 202); }
    body += 4 + lv;
  }
  if (is_value) { VSeg v; v.base1 = body; v.n0 = rs.num_rows; v._pad = 0; P.vseg[si] = v; }
  return body;
}
__device__ __forceinline__ const uint8_t* slot_base(const FParams& P, uint32_t si, int s) { return P.bases[size_t(si) * MAXC + s]; }
// cold: one widened value addressed by (row group, slot, row)
__device__ __noinline__ uint64_t fetch_val(const FParams& P, uint32_t si, int s, uint32_t row) {
  return load_kind(slot_base(P, si, s), P.kind[s], row);
}

// Time bucket of ts as the closed range [lo, hi] of timestamps that truncate to the same bucket start
// (bucket = ts / w * w with TRUNCATING division, types.rs:82-85: bucket 0 spans (-w, w)).  The range saturates at the
// ends of i64: the first and last buckets of the type hold fewer than w timestamps, and start -/+ (w - 1) must not wrap.
struct Bucket { int64_t start, lo, hi; };
__device__ __noinline__ Bucket bucket_range(int64_t ts, int64_t w) {
  constexpr int64_t kMin = INT64_MIN, kMax = INT64_MAX;
  const int64_t r = w - 1;
  Bucket b;
  b.start = ts / w * w;
  if (b.start > 0) { b.lo = b.start; b.hi = b.start > kMax - r ? kMax : b.start + r; }
  else if (b.start < 0) { b.lo = b.start < kMin + r ? kMin : b.start - r; b.hi = b.start; }
  else { b.lo = -r; b.hi = r; }
  return b;
}

// Rare path: row (si,row) has the same PK as the row after it (or is the last row of its row group).  It is dropped
// iff some LATER row of the same PK run passes the predicate (the filter runs before merge/dedup: read.rs:459-480).
__device__ __noinline__ bool later_alive_dup(const FParams& P, uint32_t si, uint32_t row) {
  uint64_t pk[MAX_PK];
  for (int k = 0; k < P.npk; k++) pk[k] = fetch_val(P, si, k, row);
  uint32_t nrows = P.sel[si].num_rows;
  uint32_t r = row + 1;
  for (;;) {
    if (r >= nrows) {
      si++;
      if (si >= *P.d_nsel) return false;
      nrows = P.sel[si].num_rows;
      r = 0;
      if (nrows == 0) continue;
    }
    for (int k = 0; k < P.npk; k++)
      if (fetch_val(P, si, k, r) != pk[k]) return false;
    bool ok = true;
    if (P.gate_slot >= 0) {                  // the conjunction of the gate column's predicates is its bit
      const uint32_t* gb = reinterpret_cast<const uint32_t*>(P.scratch + P.sel[si].scratch_off + P.bits_off);
      ok = (gb[r >> 5] >> (r & 31)) & 1u;
    }
    for (int p = 0; p < P.npred && ok; p++)
      if (P.pslot[p] != P.gate_slot) ok = op_holds(cmp_widened(fetch_val(P, si, P.pslot[p], r), P.plit[p], P.cls[P.pslot[p]]), P.pop[p]);
    if (ok) return true;
    r++;
  }
}

__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) {
  uint32_t lo = __shfl_sync(0xffffffffu, uint32_t(v), src);
  uint32_t hi = __shfl_sync(0xffffffffu, uint32_t(v >> 32), src);
  return (uint64_t(hi) << 32) | lo;
}
__device__ __forceinline__ double shfl_xor_d(double v, int m) {
  uint64_t b = uint64_t(__double_as_longlong(v));
  uint32_t lo = __shfl_xor_sync(0xffffffffu, uint32_t(b), m);
  uint32_t hi = __shfl_xor_sync(0xffffffffu, uint32_t(b >> 32), m);
  return __longlong_as_double((long long)((uint64_t(hi) << 32) | lo));
}

struct Acc {
  bool open;
  uint64_t g;
  int64_t bstart, blo, bhi;
  uint64_t cnt;
  double sum, mn, mx;
};

// Record slots are reserved 32 at a time per warp (slots = {next, end} in shared memory): one global atomic per 32 groups.
__device__ __noinline__ void emit(const FParams& P, const Acc& a, uint32_t item, uint32_t local, uint32_t* slots) {
  if (slots[0] == slots[1]) { slots[0] = atomicAdd(&P.work[1], 32u); slots[1] = slots[0] + 32u; }
  unsigned int slot = slots[0]++;
  if (slot < P.rec_cap) {
    FRec r;
    r.item = item; r.local = local; r.gkey = a.g; r.bucket = a.bstart; r.count = a.cnt; r.sum = a.sum; r.mn = a.mn; r.mx = a.mx; r._pad = 0;
    P.rec[slot] = r;
  } else atomicExch(P.err, 201);
}

// ------------------------------------------------------------------------------------------- row-group selection
// Statistics pruning on the device (DataFusion PruningPredicate, read.rs:613: CASE WHEN null_count = row_count THEN
// false ELSE <min/max rewrite> END) over the per-SST tables that live next to the SST bytes.  One block walks the row
// groups of all files in stream order and writes the compacted RgSel list — the host touches only per-FILE facts.
struct FileDev {
  const RgCol* rgcol;
  const uint32_t* rg_rows;
  uint32_t rg_base, nrg, ncols, _pad;
  const uint8_t* bytes;         // the resident file (bloom filter bitsets)
};

__global__ void __launch_bounds__(256) slot_bases_kernel(const __grid_constant__ FParams P, const uint8_t** __restrict__ bases) {
  const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t si = idx / MAXC;
  const int s = int(idx % MAXC);
  if (si >= *P.d_nsel || s >= P.nslots) return;
  bases[idx] = slot_base_chase(P, si, s);
}

// Gate-first decompression of Snappy SSTs, row-group level: after the gate column's pages are decompressed, find the
// row groups that hold a row passing the gate column's predicates; the other columns are decompressed only for those.
// The filter runs before merge and dedup (read.rs:459-480), so a row group without a passing row contributes nothing.
// It also records, per row group, how many leading rows can matter at all: everything behind the LAST row that passes the
// gate fails the filter, so the remaining columns only have to be decompressed up to there (RgSel::out_row = that row + 2:
// the row itself and its successor for the LastValue comparison).  With P.gate_bits it keeps what the scan needs of the gate column,
// one bit per row (bit r & 31 of word r >> 5, bits past the last row zero): the fused kernel's gate sweeps read those instead of the values.
// A block takes row groups blockIdx.x, blockIdx.x + gridDim.x, ..; the gate column's base of each (a chain of dependent loads through the
// resident tables) is found for 256 of them at once, one per thread, before any is tested.  Thread t tests rows t, t + 256, ..: warp w's
// ballot is bitmap word 8k + w.
template <bool W4>
__global__ void __launch_bounds__(256, 8) gate_rg_kernel(const __grid_constant__ FParams P, RgSel* __restrict__ sel, int gate_slot, uint64_t flip,
                                                      uint64_t lo, uint64_t span, uint8_t* __restrict__ flags) {
  constexpr int kRows = W4 ? 8 : 4;                        // rows per thread and batch (32 B): every load of a batch in flight before the first ballot
  __shared__ uint32_t s_last;
  __shared__ const uint8_t* s_base[256];
  const uint32_t nsel = *P.d_nsel;
  const int lane = threadIdx.x & 31;
  for (uint32_t k0 = 0; blockIdx.x + k0 * gridDim.x < nsel; k0 += 256) {
    {
      const uint32_t si = blockIdx.x + (k0 + threadIdx.x) * gridDim.x;
      if (si < nsel) s_base[threadIdx.x] = slot_base_chase(P, si, gate_slot);
    }
    for (uint32_t k = 0; k < 256; k++) {
      const uint32_t si = blockIdx.x + (k0 + k) * gridDim.x;
      if (si >= nsel) break;
      if (threadIdx.x == 0) s_last = 0;
      __syncthreads();
      const uint8_t* base = s_base[k];
      const RgSel rs = sel[si];
      const uint32_t nrows = rs.num_rows;
      uint32_t* bits = P.gate_bits ? reinterpret_cast<uint32_t*>(const_cast<uint8_t*>(P.scratch) + rs.scratch_off + P.bits_off) : nullptr;
      const bool aligned = (reinterpret_cast<uintptr_t>(base) & (W4 ? 3 : 7)) == 0;
      uint32_t last = 0;                                   // 1 + index of the last passing row seen by this thread
      const uint32_t nw = (nrows + 31) >> 5;
      for (uint32_t i0 = 0; i0 < nw * 32; i0 += kRows * 256) {
        uint64_t v[kRows];
#pragma unroll
        for (int u = 0; u < kRows; u++) {
          const uint32_t i = i0 + u * 256 + threadIdx.x;
          v[u] = 0;
          if (i < nrows) {
            if (W4) v[u] = aligned ? __ldg(reinterpret_cast<const uint32_t*>(base) + i) : ld32u(base + size_t(i) * 4);
            else v[u] = aligned ? __ldg(reinterpret_cast<const unsigned long long*>(base) + i) : ld_bytes8(base + size_t(i) * 8);
          }
        }
#pragma unroll
        for (int u = 0; u < kRows; u++) {
          const uint32_t i = i0 + u * 256 + threadIdx.x;
          const bool pass = i < nrows && (W4 ? (uint32_t(v[u]) ^ uint32_t(flip)) - uint32_t(lo) <= uint32_t(span) : (v[u] ^ flip) - lo <= span);
          if (pass) last = i + 1;
          const uint32_t b = __ballot_sync(0xffffffffu, pass);
          if (bits && lane == 0 && (i >> 5) < nw) bits[i >> 5] = b;
        }
      }
      for (int d = 16; d > 0; d >>= 1) { const uint32_t o = __shfl_down_sync(0xffffffffu, last, d); last = o > last ? o : last; }
      if (lane == 0 && last) atomicMax(&s_last, last);
      __syncthreads();
      if (threadIdx.x == 0) {
        const uint32_t l = s_last;
        flags[si] = l ? 1 : 0;
        sel[si].out_row = l ? (l + 1 < nrows ? l + 1 : nrows) : 0;
      }
    }
    __syncthreads();                                       // every thread is done with s_base before the next 256 are found
  }
}

// one block: stable compaction of the selected row groups by flag (RgSel carries its scratch offset along).
// lpt (optional): the compacted row groups' indices ordered by descending out_row = descending decompression work of the
// partially decoded pages.  One warp decodes one page and a page is serial, so the decompression stage ends when the warp with
// the longest total finishes: handing out the longest pages first (LPT) lets the short ones fill the tail.
__global__ void __launch_bounds__(1024) compact_sel_kernel(const RgSel* __restrict__ in, const uint8_t* __restrict__ flags, uint32_t* d_nsel,
                                                           RgSel* __restrict__ out, uint32_t* __restrict__ lpt) {
  __shared__ uint32_t s_w[1024 / 32 + 1];
  __shared__ uint32_t s_bin[1024];
  __shared__ uint32_t s_max;
  const uint32_t n = *d_nsel;
  const uint32_t per = (n + 1023u) / 1024u;
  const uint32_t lo = threadIdx.x * per;
  const uint32_t hi = lo + per < n ? lo + per : n;
  uint32_t cnt = 0;
  for (uint32_t i = lo; i < hi; i++) cnt += flags[i] != 0;
  s_bin[threadIdx.x] = 0;
  if (threadIdx.x == 0) s_max = 0;
  uint32_t m;
  uint32_t pos = block_excl_scan<1024>(cnt, &m, s_w);
  uint32_t mx = 0;
  for (uint32_t i = lo; i < hi; i++)
    if (flags[i]) { out[pos++] = in[i]; mx = in[i].out_row > mx ? in[i].out_row : mx; }
  if (lpt) {
    // counting sort of the compacted list by out_row, descending (1024 bins over [0, max]; order inside a bin is arbitrary)
    if (mx) atomicMax(&s_max, mx);
    __syncthreads();
    int shift = 0;
    while ((s_max >> shift) > 1023u) shift++;
    const uint32_t per2 = (m + 1023u) / 1024u;
    const uint32_t lo2 = threadIdx.x * per2, hi2 = lo2 + per2 < m ? lo2 + per2 : m;
    for (uint32_t i = lo2; i < hi2; i++) atomicAdd(&s_bin[1023u - (out[i].out_row >> shift)], 1u);
    __syncthreads();
    uint32_t nbin;
    const uint32_t start = block_excl_scan<1024>(s_bin[threadIdx.x], &nbin, s_w);
    s_bin[threadIdx.x] = start;                                 // exclusive start of this bin
    __syncthreads();
    for (uint32_t i = lo2; i < hi2; i++) lpt[atomicAdd(&s_bin[1023u - (out[i].out_row >> shift)], 1u)] = i;
  }
  __syncthreads();
  if (threadIdx.x == 0) *d_nsel = m;
}

// phase 1: one thread per row group, all blocks in parallel: keep flag (0/1) + rows.  prune: bit 0 statistics, bit 1 bloom filters
__global__ void __launch_bounds__(256) prune_rgs_kernel(const __grid_constant__ FParams P, const FileDev* __restrict__ files, int nfiles,
                                                        uint32_t total_rgs, int prune, uint32_t* __restrict__ keep_rows) {
  const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total_rgs) return;
  uint32_t f = 0;
  while (f + 1 < uint32_t(nfiles) && idx >= files[f + 1].rg_base) f++;
  const FileDev fd = files[f];
  const uint32_t rg = idx - fd.rg_base;
  const uint32_t rows = fd.rg_rows[rg];
  uint32_t keep = rows > 0;
  if (keep && prune) {
    const RgCol* rc = fd.rgcol + size_t(rg) * fd.ncols;
    for (int p = 0; p < P.npred && keep; p++) {
      const RgCol c = rc[P.pcol[p]];
      if (c.null_all) { keep = 0; break; }
      if (c.has_minmax && !minmax_may_match(c.mn, c.mx, P.plit[p], P.pop[p], P.pcls[p])) keep = 0;
      // then the chunk's bloom filter (prune bit 1; transient files list no filter: the host probed them)
      else if ((prune & 2) && P.pbloom[p] && c.bloom_blocks && !bloom::may_contain(fd.bytes + c.bloom_off, c.bloom_blocks, P.phash[p])) keep = 0;
    }
  }
  keep_rows[idx] = keep ? rows : 0;             // rows > 0 doubles as the keep flag
}

// phase 2: one block compacts the kept row groups in stream order (coalesced reads of keep_rows)
__global__ void __launch_bounds__(1024) select_rgs_kernel(const FileDev* __restrict__ files, int nfiles, uint32_t total_rgs,
                                                          const uint32_t* keep_rows, RgSel* __restrict__ sel, uint32_t* d_nsel,
                                                          unsigned long long* counters, uint32_t smem_words, uint64_t scratch_per_rg) {
  // one block; every thread owns a contiguous chunk of row groups: count, ONE block-wide scan, write.  The keep flags are
  // staged in shared memory with coalesced loads first (smem_words == 0: too many row groups, read them in place).
  extern __shared__ uint32_t s_keep[];
  __shared__ uint32_t s_w[1024 / 32 + 1];
  if (smem_words) {
    for (uint32_t i = threadIdx.x; i < total_rgs; i += 1024) s_keep[i] = keep_rows[i];
    __syncthreads();
    keep_rows = s_keep;
  }
  const uint32_t per = (total_rgs + 1023u) / 1024u;
  const uint32_t lo = threadIdx.x * per;
  const uint32_t hi = lo + per < total_rgs ? lo + per : total_rgs;
  uint32_t cnt = 0;
  unsigned long long rows_sel = 0;
  for (uint32_t i = lo; i < hi; i++) { const uint32_t r = keep_rows[i]; cnt += r > 0; rows_sel += r; }
  uint32_t nsel;
  uint32_t pos = block_excl_scan<1024>(cnt, &nsel, s_w);
  if (cnt) {
    uint32_t f = 0;
    for (uint32_t i = lo; i < hi; i++) {
      const uint32_t rows = keep_rows[i];
      if (rows == 0) continue;
      while (f + 1 < uint32_t(nfiles) && i >= files[f + 1].rg_base) f++;
      RgSel r;
      r.sst = f; r.rg = i - files[f].rg_base; r.out_row = 0; r.num_rows = rows; r.scratch_off = uint64_t(pos) * scratch_per_rg;
      sel[pos++] = r;
    }
  }
  for (int d = 16; d > 0; d >>= 1) rows_sel += __shfl_down_sync(0xffffffffu, rows_sel, d);
  if ((threadIdx.x & 31) == 0 && rows_sel) atomicAdd(&counters[2], rows_sel);
  if (threadIdx.x == 0) *d_nsel = nsel;
}

// ------------------------------------------------------------------------------------------------ item boundaries
// Work items are sub-ranges of row groups.  A group (key-run) must be summed by ONE warp in stream order, so every
// nominal boundary is moved forward to the next row that starts a new key-run: item j = [adj[j], adj[j+1]).
// One warp per boundary; the run end is located by 32-way probing (keys are sorted, so "differs from the key at the
// boundary" is monotone along the stream): 3 rounds cover a 8192-row group.
struct KeyRef { uint64_t g; int64_t lo, hi; };

__device__ __forceinline__ uint64_t pack_pos(uint32_t si, uint32_t row) { return (uint64_t(si) << 32) | row; }

// One boundary search, advanced one probing round at a time so that a warp can interleave several of them
// (their dependent load chains overlap: the kernel is pure latency).
template <bool HAS_TS>
struct BoundSearch {
  uint32_t j, si, row, L, H, ans;
  KeyRef k;
  const uint8_t *b0, *b1;
  bool done, found;

  __device__ __forceinline__ void finish(uint64_t* adj, uint64_t v, int lane) { if (lane == 0) adj[j] = v; done = true; }

  __device__ __forceinline__ void open_rg(const FParams& P) {
    b0 = P.has_group ? slot_base(P, si, 0) : nullptr;
    b1 = HAS_TS ? slot_base(P, si, 1) : nullptr;
    L = row;
    H = P.sel[si].num_rows;
    found = false;
    ans = H;
  }

  __device__ __forceinline__ void init(const FParams& P, uint32_t jj, uint32_t nsel, uint32_t nitems, uint64_t* adj, int lane) {
    j = jj;
    done = false;
    if (j > nitems) { done = true; return; }
    if (j == nitems) { finish(adj, pack_pos(nsel, 0), lane); return; }
    si = j / P.split;
    const uint32_t w = j % P.split;
    const uint32_t n = P.sel[si].num_rows;
    const uint32_t sr = (((n + P.split - 1) / P.split) + 31u) & ~31u;
    row = w * sr;
    if (row >= n) { si++; row = 0; }                        // empty sub-range: same boundary as the next row group
    if (si >= nsel) { finish(adj, pack_pos(nsel, 0), lane); return; }
    if (P.global_mode || (si == 0 && row == 0)) { finish(adj, pack_pos(si, row), lane); return; }
    uint32_t psi = si, prow = row;                          // key of the row just before the nominal boundary
    if (prow == 0) { psi--; prow = P.sel[psi].num_rows - 1; } else prow--;
    k.g = P.has_group ? fetch_val(P, psi, 0, prow) : 0;
    k.lo = 0; k.hi = 0;
    if (HAS_TS) { Bucket b = bucket_range(int64_t(fetch_val(P, psi, 1, prow)), P.window_ms); k.lo = b.lo; k.hi = b.hi; }
    open_rg(P);
  }

  // probe position of this lane in the current window [L, H) (32 chunks; the lane looks at the last row of its chunk)
  __device__ __forceinline__ uint32_t probe_pos(int lane, uint32_t* step) const {
    const uint32_t span = H - L;
    *step = (span + 31) / 32;
    uint32_t p = L + (uint32_t(lane) + 1) * *step - 1;
    return p >= H ? H - 1 : p;
  }

  __device__ __forceinline__ void advance(const FParams& P, unsigned m, uint32_t step, uint32_t nsel, uint64_t* adj, int lane) {
    if (m == 0) L = H;                                      // the whole window continues the run
    else {
      const int f = __ffs(m) - 1;
      uint32_t pf = L + (uint32_t(f) + 1) * step - 1;
      if (pf >= H) pf = H - 1;
      found = true;
      ans = pf;
      if (step == 1) L = H;                                 // exact
      else { L = L + uint32_t(f) * step; H = pf; }          // rows [L, pf) still unknown; pf differs
    }
    if (L >= H) {
      if (found) { finish(adj, pack_pos(si, ans), lane); return; }
      si++;                                                 // the run covers the rest of this row group
      row = 0;
      if (si >= nsel) { finish(adj, pack_pos(nsel, 0), lane); return; }
      open_rg(P);
    }
  }
};

constexpr int kBoundsPerWarp = 4;

template <bool HAS_TS>
__global__ void __launch_bounds__(256) item_bounds_kernel(const __grid_constant__ FParams P, uint64_t* __restrict__ adj) {
  const int lane = threadIdx.x & 31;
  const uint32_t nsel = *P.d_nsel;
  const uint32_t nitems = nsel * P.split;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  BoundSearch<HAS_TS> bs[kBoundsPerWarp];
#pragma unroll
  for (int i = 0; i < kBoundsPerWarp; i++) bs[i].init(P, warp * kBoundsPerWarp + i, nsel, nitems, adj, lane);
  for (;;) {
    bool any = false;
    uint32_t step[kBoundsPerWarp];
    uint64_t v0[kBoundsPerWarp], v1[kBoundsPerWarp];
#pragma unroll
    for (int i = 0; i < kBoundsPerWarp; i++) {              // issue every search's probe loads first
      v0[i] = 0; v1[i] = 0; step[i] = 1;
      if (!bs[i].done) {
        any = true;
        const uint32_t p = bs[i].probe_pos(lane, &step[i]);
        if (P.has_group) v0[i] = load_kind(bs[i].b0, P.kind[0], p);
        if (HAS_TS) v1[i] = load_kind(bs[i].b1, P.kind[1], p);
      }
    }
    if (!any) break;
#pragma unroll
    for (int i = 0; i < kBoundsPerWarp; i++) {
      if (!bs[i].done) {
        bool ne = (P.has_group && v0[i] != bs[i].k.g) || (HAS_TS && (int64_t(v1[i]) < bs[i].k.lo || int64_t(v1[i]) > bs[i].k.hi));
        const unsigned m = __ballot_sync(0xffffffffu, ne);
        bs[i].advance(P, m, step[i], nsel, adj, lane);
      }
    }
  }
}

// Survivors of one slice, fast path: they all extend the open group.  count by popc, min/max by a warp butterfly that
// equals the sequential rule (see walk_slice); the f64 sum is a strictly sequential chain in stream order.  With many survivors the values go through
// shared memory (non-survivors contribute +0.0, which is exact because the running sum starts at +0.0 and can never
// be -0.0): 32 x (LDS + DADD) straight-line instead of a 12-instruction loop per survivor.
__device__ __forceinline__ double seq_sum_slice(double sum, unsigned keep_mask, bool keep, double v, double* s_vals, int lane) {
  if (__popc(keep_mask) >= 8) {
    __syncwarp();
    s_vals[lane] = keep ? v : 0.0;
    __syncwarp();
#pragma unroll
    for (int l = 0; l < 32; l++) sum += s_vals[l];
    return sum;
  }
  uint64_t vb = uint64_t(__double_as_longlong(v));
  while (keep_mask) {
    int l = __ffs(keep_mask) - 1;
    keep_mask &= keep_mask - 1;
    sum += __longlong_as_double((long long)shfl64(vb, l));
  }
  return sum;
}

template <bool HAS_TS>
__device__ __noinline__ void walk_slice(const FParams& P, Acc& acc, uint32_t& local, uint32_t item, unsigned keep_mask, bool keep, uint64_t g,
                                        int64_t ts, double v, double* s_vals, uint32_t* slots, int lane) {
  const double kInf = __longlong_as_double(0x7ff0000000000000LL);
  const bool has_val = P.value_slot >= 0;
  bool ext = keep && acc.open && (!P.has_group || g == acc.g) && (!HAS_TS || (ts >= acc.blo && ts <= acc.bhi));
  if (__ballot_sync(0xffffffffu, ext) == keep_mask) {
    acc.cnt += __popc(keep_mask);
    if (has_val) {
      // The sequential rule (`x < mn` / `x > mx` over the survivors in stream order = lane order, on a group that already
      // holds its first value) as a butterfly: a NaN is never taken, so it enters as the identity, and on a tie the lower
      // lanes win, which decides between -0.0 and +0.0.  Distances grow, so that every lane's partial covers a contiguous
      // range of lanes: at distance m the lanes with bit m set hold the later of the two ranges.
      const bool num = keep && v == v;
      double mn = num ? v : kInf, mx = num ? v : -kInf;
#pragma unroll
      for (int m = 1; m < 32; m <<= 1) {
        const double a = shfl_xor_d(mn, m), b = shfl_xor_d(mx, m);
        const bool later = (lane & m) != 0;
        mn = (later ? a <= mn : a < mn) ? a : mn;
        mx = (later ? b >= mx : b > mx) ? b : mx;
      }
      acc.mn = mn < acc.mn ? mn : acc.mn;
      acc.mx = mx > acc.mx ? mx : acc.mx;
      acc.sum = seq_sum_slice(acc.sum, keep_mask, keep, v, s_vals, lane);
    }
    return;
  }
  uint64_t vb = uint64_t(__double_as_longlong(v));
  while (keep_mask) {
    int l = __ffs(keep_mask) - 1;
    keep_mask &= keep_mask - 1;
    uint64_t kg = P.has_group ? shfl64(g, l) : 0;
    int64_t kt = HAS_TS ? int64_t(shfl64(uint64_t(ts), l)) : 0;
    if (!acc.open || kg != acc.g || (HAS_TS && (kt < acc.blo || kt > acc.bhi))) {
      if (acc.open) { if (lane == 0) emit(P, acc, item, local, slots); local++; }
      acc.open = true; acc.g = kg; acc.cnt = 0; acc.sum = 0.0; acc.mn = kInf; acc.mx = -kInf;
      if (HAS_TS) { Bucket b = bucket_range(kt, P.window_ms); acc.bstart = b.start; acc.blo = b.lo; acc.bhi = b.hi; }
      else { acc.bstart = 0; acc.blo = 0; acc.bhi = 0; }
    }
    acc.cnt++;
    if (has_val) {
      double x = __longlong_as_double((long long)shfl64(vb, l));
      acc.sum += x;
      if (acc.cnt == 1 || x < acc.mn) acc.mn = x;
      if (acc.cnt == 1 || x > acc.mx) acc.mx = x;
    }
  }
}

__device__ __forceinline__ double to_double_kind(uint64_t raw, uint32_t kind, uint32_t cls) {
  uint64_t wv = widen_kind(raw, kind);
  return cls == C_FLOAT ? __longlong_as_double((long long)wv) : (cls == C_SIGNED ? double(int64_t(wv)) : double(wv));
}

__device__ __forceinline__ uint64_t ld8(const uint8_t* q, uint32_t sh, uint32_t i) {
  const uint64_t* p = reinterpret_cast<const uint64_t*>(q) + i;
  uint64_t lo = __ldg(p), hi = __ldg(p + 1);
  uint32_t w0 = uint32_t(lo), w1 = uint32_t(lo >> 32), w2 = uint32_t(hi), w3 = uint32_t(hi >> 32);
  const bool up = (sh & 32u) != 0;
  const uint32_t s = sh & 31u;
  uint32_t a = up ? w1 : w0, b = up ? w2 : w1, c = up ? w3 : w2;
  return (uint64_t(__funnelshift_r(b, c, s)) << 32) | __funnelshift_r(a, b, s);
}
__device__ __forceinline__ uint32_t ld4(const uint8_t* q, uint32_t sh, uint32_t i) {
  const uint32_t* p = reinterpret_cast<const uint32_t*>(q) + i;
  uint32_t lo = __ldg(p), hi = __ldg(p + 1);
  return __funnelshift_r(lo, hi, sh);
}

// Cursor of the value column inside the current row group.  Normally one contiguous array (split = all rows); a stored
// Snappy page is read in place as two arrays: rows [0, split) behind q0, rows [split, ..) behind q1.
struct VCur {
  const uint8_t *q0, *q1;    // bases rounded down to the value width
  uint32_t s0, s1;           // bit shifts of the values inside their aligned words
  uint32_t split;
};
__device__ __forceinline__ uint64_t ldv(const VCur& V, bool v8, uint32_t i) {
  const bool a = i < V.split;
  const uint8_t* q = a ? V.q0 : V.q1;
  const uint32_t sh = a ? V.s0 : V.s1;
  const uint32_t j = a ? i : i - V.split;
  return v8 ? ld8(q, sh, j) : uint64_t(ld4(q, sh, j));
}

// Per-column constants of the hot columns, held in registers across the whole item.
template <int NH>
struct Hot {
  const uint8_t* q[NH];      // value base rounded down to the column's word size (changes with the row group)
  uint32_t sh[NH];           // bit shift of the values inside their aligned words
  uint64_t flip[NH], lo[NH], span[NH];
  bool haspred[NH];
  const uint32_t* gbits;     // gated kernels: the row group's gate bitmap (FParams::gate_bits), else nullptr
};

// One block = kU slices of 32 rows.  Phase 1 issues every load of the block as straight-line code: kU*NH*2 loads per
// lane in flight.  Phase 2 walks the slices in stream order; everything beyond the interval tests runs only when a
// slice has survivors.  Only `dense` is a compile-time choice (two copies per kernel); clamping / masking and the
// prefetch are runtime, warp-uniform choices: the kernel's instruction footprint matters — with four specialised copies
// a fifth of the stall samples were instruction-cache misses.
//   X      bit k set => extra hot column 2+k is a 4-byte column (pk0 / pk1 are always 8-byte here)
//   dense  most rows survive: the value column and the halo row are loaded with the block, not per survivor
//   pf     prefetch the block two iterations ahead into L2 (sequential walks only)
// The block may extend past `lim` (end of the item or of the row group): indices are clamped, lanes masked.
template <int kU, int NH, int X, bool HAS_TS, bool dense>
__device__ __forceinline__ uint32_t process_block(const FParams& P, const Hot<NH>& H, const VCur& V, Acc& acc, uint32_t& local,
                                                  uint32_t& n_alive, uint32_t& n_keep, uint32_t& n_full, uint32_t item, uint32_t csi, uint32_t row,
                                                  uint32_t lim, uint32_t nrows, bool pf, double* s_vals, uint32_t* slots, int lane) {
  uint64_t hv[kU][NH];
  uint64_t vv[kU];
  uint64_t halo[2] = {0, 0};
  const uint32_t last = nrows - 1;
  if (pf) {
    // pull the hot columns of the block two blocks ahead into L2: one 128-byte line per lane
    const uint32_t prow = row + 2 * 32 * kU;
#pragma unroll
    for (int h = 0; h < NH; h++) {
      const bool w4 = h >= 2 && ((X >> (h - 2)) & 1);
      const uint32_t per_line = w4 ? 32u : 16u;                 // rows per 128-byte line
      const uint32_t r = prow + uint32_t(lane) * per_line;
      if (uint32_t(lane) <= (32u * kU) / per_line && r < nrows)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(H.q[h] + size_t(r) * (w4 ? 4 : 8)));
    }
  }
  n_full += lim - row < 32u * kU ? lim - row : 32u * kU;
#pragma unroll
  for (int u = 0; u < kU; u++) {
    uint32_t i = row + u * 32 + lane;
    i = i < last ? i : last;
#pragma unroll
    for (int h = 0; h < NH; h++) {
      const bool w4 = h >= 2 && ((X >> (h - 2)) & 1);
      if (h == NH - 1 && h >= 2 && H.gbits) { hv[u][h] = __ldg(H.gbits + (i >> 5)); continue; }   // a gate that is not a key: its bit word
      hv[u][h] = w4 ? uint64_t(ld4(H.q[h], H.sh[h], i)) : ld8(H.q[h], H.sh[h], i);
    }
  }
  const bool v8 = P.value_slot >= 0 && P.kind[P.value_slot] == K_RAW64;
  if (dense) {
    uint32_t i = row + kU * 32;
    i = i < last ? i : last;
    halo[0] = ld8(H.q[0], H.sh[0], i);
    halo[1] = ld8(H.q[1], H.sh[1], i);
#pragma unroll
    for (int u = 0; u < kU; u++) {
      uint32_t i2 = row + u * 32 + lane;
      i2 = i2 < last ? i2 : last;
      vv[u] = ldv(V, v8, i2);
    }
  }
  uint32_t kept_in_block = 0;
#pragma unroll
  for (int u = 0; u < kU; u++) {
    const uint32_t i = row + u * 32 + lane;
    bool alive = i < lim;
#pragma unroll
    for (int h = 0; h < NH; h++) {
      const bool w4 = h >= 2 && ((X >> (h - 2)) & 1);
      if (h == NH - 1 && h >= 2 && H.gbits) alive = alive && ((uint32_t(hv[u][h]) >> (i & 31)) & 1u);
      else if (H.haspred[h]) {                         // uniform
        if (w4) alive = alive && ((uint32_t(hv[u][h]) ^ uint32_t(H.flip[h])) - uint32_t(H.lo[h]) <= uint32_t(H.span[h]));
        else alive = alive && ((hv[u][h] ^ H.flip[h]) - H.lo[h] <= H.span[h]);
      }
    }
    const unsigned alive_mask = __ballot_sync(0xffffffffu, alive);
    if (alive_mask == 0) continue;
    // dedup: compare with the NEXT row of the stream (LastValue keeps the last row of a PK run).  The next row's
    // pk0 / pk1 come from the neighbouring lane (or the next slice / the halo row), not from memory.
    uint64_t n0 = shfl64(hv[u][0], (lane + 1) & 31), n1 = shfl64(hv[u][1], (lane + 1) & 31);
    if (u + 1 < kU) {
      uint64_t f0 = shfl64(hv[u + 1 < kU ? u + 1 : u][0], 0), f1 = shfl64(hv[u + 1 < kU ? u + 1 : u][1], 0);
      if (lane == 31) { n0 = f0; n1 = f1; }
    } else {
      if (!dense && (alive_mask >> 31)) {              // sparse blocks fetch the halo row only when lane 31 survives
        uint32_t ih = row + kU * 32;
        ih = ih < last ? ih : last;
        halo[0] = ld8(H.q[0], H.sh[0], ih);
        halo[1] = ld8(H.q[1], H.sh[1], ih);
      }
      if (lane == 31) { n0 = halo[0]; n1 = halo[1]; }
    }
    bool keep = alive;
    if (alive) {
      bool same = true;
      if (i + 1 < nrows) {
        same = n0 == hv[u][0] && n1 == hv[u][1];
        for (int k = 2; k < P.npk && same; k++) same = fetch_val(P, csi, k, i + 1) == fetch_val(P, csi, k, i);
      }
      if (same && (i + 1 < nrows || csi + 1 < *P.d_nsel)) keep = !later_alive_dup(P, csi, i);
    }
    const unsigned keep_mask = __ballot_sync(0xffffffffu, keep);
    n_alive += __popc(alive_mask);
    n_keep += __popc(keep_mask);
    kept_in_block += __popc(keep_mask);
    if (!P.global_mode && keep_mask) {
      double v = 0.0;
      if (P.value_slot >= 0) {
        uint64_t raw = vv[u];
        if (!dense) raw = keep ? ldv(V, v8, i) : 0ull;
        v = to_double_kind(raw, P.kind[P.value_slot], P.cls[P.value_slot]);
      }
      walk_slice<HAS_TS>(P, acc, local, item, keep_mask, keep, hv[u][0], int64_t(hv[u][1]), v, s_vals, slots, lane);
    }
  }
  return kept_in_block;
}

// Late materialisation: the LAST hot column (the planner puts the narrowest predicate column there) is the gate.  One
// sweep tests the gate values of kGS consecutive slices (1-2 KB per warp in flight) and returns one bit per 32*kU-row
// block that holds a passing row; only those blocks run the full block code (which reads the other columns).
// The sweep may extend past `lim`: indices are clamped to the row group, rows >= lim masked.
// Gate bits: lane u < kGS takes slice u's 32 bits (a funnel of two words: items start at key-run boundaries, not at
// multiples of 32).
template <int kU, int NH, int X, int kGS>
__device__ __forceinline__ uint32_t gate_sweep(const Hot<NH>& H, uint32_t row, uint32_t lim, uint32_t nrows, int lane) {
  constexpr int G = NH - 1;
  constexpr bool w4 = G >= 2 && ((X >> (G - 2)) & 1);
  if (H.gbits) {
    const uint32_t* bw = H.gbits;
    const uint32_t nw = (nrows + 31) >> 5;
    uint32_t sb = 0;
    const uint32_t r = row + uint32_t(lane) * 32u;
    if (lane < kGS && r < lim) {
      const uint32_t w = r >> 5;
      const uint32_t a = __ldg(bw + w), b = w + 1 < nw ? __ldg(bw + w + 1) : 0u;
      sb = __funnelshift_r(a, b, r & 31);
      if (lim - r < 32) sb &= (1u << (lim - r)) - 1;
    }
    const unsigned m = __ballot_sync(0xffffffffu, sb != 0);
    uint32_t bm = 0;
#pragma unroll
    for (int u = 0; u < kGS; u++)
      if ((m >> u) & 1u) bm |= 1u << (u / kU);
    return bm;
  }
  {                                                         // next-but-one sweep's gate bytes into L2, one line per lane
    constexpr uint32_t per_line = w4 ? 32u : 16u;
    const uint32_t r = row + 2u * 32u * kGS + uint32_t(lane) * per_line;
    if (uint32_t(lane) < (32u * kGS) / per_line + 1 && r < nrows)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(H.q[G] + size_t(r) * (w4 ? 4 : 8)));
  }
  const uint32_t last = nrows - 1;
  uint64_t gv[kGS];
#pragma unroll
  for (int u = 0; u < kGS; u++) {
    uint32_t i = row + u * 32 + lane;
    i = i < last ? i : last;
    gv[u] = w4 ? uint64_t(ld4(H.q[G], H.sh[G], i)) : ld8(H.q[G], H.sh[G], i);
  }
  uint32_t bm = 0;
#pragma unroll
  for (int u = 0; u < kGS; u++) {
    bool pass = w4 ? ((uint32_t(gv[u]) ^ uint32_t(H.flip[G])) - uint32_t(H.lo[G]) <= uint32_t(H.span[G]))
                   : ((gv[u] ^ H.flip[G]) - H.lo[G] <= H.span[G]);
    pass = pass && (row + u * 32 + lane < lim);
    if (__ballot_sync(0xffffffffu, pass)) bm |= 1u << (u / kU);
  }
  return bm;
}

// After a sweep: start pulling the other columns (and the value column) of the blocks that will be materialised into L2,
// all at once, so that the block code that follows finds them there instead of paying one DRAM round trip per block.
template <int kU, int NH, int X, int kGS>
__device__ __forceinline__ void prefetch_blocks(const Hot<NH>& H, const uint8_t* vq, bool has_val, bool v8, uint32_t bm, uint32_t row,
                                                uint32_t nrows, int lane) {
#pragma unroll
  for (int h = 0; h < NH - 1; h++) {
    const bool w4 = h >= 2 && ((X >> (h - 2)) & 1);
    const uint32_t off = uint32_t(lane) * (w4 ? 32u : 16u);          // first row of this lane's 128-byte line
    uint32_t blk = off / (32u * kU);
    blk = blk < uint32_t(kGS / kU) ? blk : uint32_t(kGS / kU) - 1;   // (one extra line: the values are not line aligned)
    if (off <= 32u * kGS && ((bm >> blk) & 1u) && row + off < nrows)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(H.q[h] + size_t(row + off) * (w4 ? 4 : 8)));
  }
  if (has_val) {
    const uint32_t off = uint32_t(lane) * (v8 ? 16u : 32u);
    uint32_t blk = off / (32u * kU);
    blk = blk < uint32_t(kGS / kU) ? blk : uint32_t(kGS / kU) - 1;
    if (off <= 32u * kGS && ((bm >> blk) & 1u) && row + off < nrows)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(vq + size_t(row + off) * (v8 ? 8 : 4)));
  }
}

// kU = slices whose loads are issued together; NH = hot columns (pk0, pk1, + predicate columns) loaded for every row
template <int kU, int kMinBlocks, int NH, int X, bool HAS_TS, bool GATED>
__global__ void __launch_bounds__(kWarpsPerCta * 32, kMinBlocks) fused_scan_kernel(const __grid_constant__ FParams P,
                                                                                    const uint64_t* __restrict__ adj) {
  __shared__ double s_vals_all[kWarpsPerCta][32];
  __shared__ uint32_t s_slots[kWarpsPerCta][2];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double* s_vals = s_vals_all[wid];
  uint32_t* slots = s_slots[wid];
  if (lane == 0) { slots[0] = 0; slots[1] = 0; }
  __syncwarp();
  const uint32_t nsel = *P.d_nsel;
  const uint32_t nitems = nsel * P.split;
  constexpr int kGS = ((NH - 1) >= 2 && ((X >> (NH - 3)) & 1)) ? 16 : 8;   // slices per gate sweep: 16 x 4-byte or 8 x 8-byte values per lane
  const double kInf = __longlong_as_double(0x7ff0000000000000LL);
  Hot<NH> H;
#pragma unroll
  for (int h = 0; h < NH; h++) {
    H.flip[h] = P.hot_flip[h]; H.lo[h] = P.hot_lo[h]; H.span[h] = P.hot_span[h]; H.haspred[h] = P.hot_haspred[h] != 0;
    H.q[h] = nullptr; H.sh[h] = 0;
  }
  VCur V;
  V.q0 = nullptr; V.q1 = nullptr; V.s0 = 0; V.s1 = 0; V.split = 0xffffffffu;
  H.gbits = nullptr;
  auto set_cursor = [&](uint32_t si) {
    // every lane derives the same pointers (loads broadcast); keeps them in registers until the next row group
    if (GATED && P.gate_bits) H.gbits = reinterpret_cast<const uint32_t*>(P.scratch + P.sel[si].scratch_off + P.bits_off);
#pragma unroll
    for (int h = 0; h < NH; h++) {
      const uintptr_t a = reinterpret_cast<uintptr_t>(slot_base(P, si, P.hot_slot[h]));
      const bool w4 = h >= 2 && ((X >> (h - 2)) & 1);
      const uintptr_t m = w4 ? 3 : 7;
      H.q[h] = reinterpret_cast<const uint8_t*>(a & ~m);
      H.sh[h] = uint32_t(a & m) * 8;
    }
    if (P.value_slot >= 0) {
      const uintptr_t a = reinterpret_cast<uintptr_t>(slot_base(P, si, P.value_slot));
      const uintptr_t m = P.kind[P.value_slot] == K_RAW64 ? 7 : 3;
      V.q0 = reinterpret_cast<const uint8_t*>(a & ~m);
      V.s0 = uint32_t(a & m) * 8;
      if (P.value_stored) {
        const VSeg vg = P.vseg[si];
        const uintptr_t b = reinterpret_cast<uintptr_t>(vg.base1);
        V.q1 = reinterpret_cast<const uint8_t*>(b & ~m);
        V.s1 = uint32_t(b & m) * 8;
        V.split = vg.n0;
      }
    }
  };
  for (;;) {
    uint32_t item = 0;
    if (lane == 0) item = atomicAdd(&P.work[0], 1u);
    item = __shfl_sync(0xffffffffu, item, 0);
    if (item >= nitems) {
      // hand back the unused part of this warp's last reservation as invalid records
      if (lane == 0) for (uint32_t sl = slots[0]; sl < slots[1]; sl++) if (sl < P.rec_cap) P.rec[sl].item = 0xffffffffu;
      return;
    }
    const uint64_t beg = adj[item], end = adj[item + 1];
    uint32_t csi = uint32_t(beg >> 32), row = uint32_t(beg);
    const uint32_t esi = uint32_t(end >> 32), erow = uint32_t(end);
    uint32_t local = 0, n_alive = 0, n_keep = 0, n_full = 0;
    if (beg < end) {
      Acc acc;
      acc.open = false; acc.g = 0; acc.bstart = 0; acc.blo = 0; acc.bhi = 0; acc.cnt = 0; acc.sum = 0.0; acc.mn = kInf; acc.mx = -kInf;
      bool dense = false;                 // most rows survive: load the value column with the block, not per survivor
      uint32_t bm = 0, sweep_kept = 0;    // gated kernels: blocks of the current sweep still to be materialised
      uint32_t nrows = P.sel[csi].num_rows;
      set_cursor(csi);
      for (;;) {
        if (row >= nrows) {
          csi++;
          row = 0;
          if (csi > esi || (csi == esi && erow == 0) || csi >= nsel) break;
          nrows = P.sel[csi].num_rows;
          set_cursor(csi);
        }
        const uint32_t lim = csi == esi ? erow : nrows;
        if (row >= lim) break;
        if (dense) {
          // dense stretch (>= 1/4 of the rows survive): everything is needed, value column loaded with the block
          const uint32_t kept = process_block<kU, NH, X, HAS_TS, true>(P, H, V, acc, local, n_alive, n_keep, n_full, item, csi, row, lim, nrows,
                                                                      true, s_vals, slots, lane);
          dense = kept >= 32u * kU / 4;
          row += 32 * kU;
          continue;
        }
        uint32_t brow = row;
        if (GATED) {
          if (bm == 0) {
            // late materialisation, coarse step: test the gate column of kGS slices, then run the block code only on the
            // 32*kU-row blocks that hold a passing row
            bm = gate_sweep<kU, NH, X, kGS>(H, row, lim, nrows, lane);
            sweep_kept = 0;
            if (bm == 0) { row += 32u * kGS; continue; }
            prefetch_blocks<kU, NH, X, kGS>(H, V.q0, P.value_slot >= 0, P.value_slot >= 0 && P.kind[P.value_slot] == K_RAW64, bm, row, nrows, lane);
          }
          brow = row + (__ffs(bm) - 1) * 32u * kU;
          bm &= bm - 1;
        }
        const uint32_t kept = process_block<kU, NH, X, HAS_TS, false>(P, H, V, acc, local, n_alive, n_keep, n_full, item, csi, brow, lim, nrows,
                                                                     !GATED, s_vals, slots, lane);
        if (GATED) {
          sweep_kept += kept;
          if (bm == 0) {                              // sweep finished
            const uint32_t swept = lim - row < 32u * kGS ? lim - row : 32u * kGS;
            dense = P.value_slot >= 0 && sweep_kept >= swept / 4;
            row += 32u * kGS;
          }
        } else {
          dense = P.value_slot >= 0 && kept >= 32u * kU / 4;
          row += 32 * kU;
        }
      }
      if (acc.open) { if (lane == 0) emit(P, acc, item, local, slots); local++; }
    }
    if (lane == 0) {
      P.item_cnt[item] = local;
      if (n_alive) atomicAdd(&P.counters[0], (unsigned long long)n_alive);
      if (n_keep) atomicAdd(&P.counters[1], (unsigned long long)n_keep);
      if (n_full) atomicAdd(&P.counters[3], (unsigned long long)n_full);
    }
  }
}

template <int kU, int kMinBlocks>
void launch_fused(int nhot, int xmask, bool has_ts, bool gated, int ctas, cudaStream_t s, const FParams& P, const uint64_t* adj) {
#define HG_LAUNCH2(NH, XM, TS)                                                                                           \
  do {                                                                                                                   \
    if (gated) fused_scan_kernel<kU, kMinBlocks, NH, XM, TS, true><<<ctas, kWarpsPerCta * 32, 0, s>>>(P, adj);      \
    else fused_scan_kernel<kU, kMinBlocks, NH, XM, TS, false><<<ctas, kWarpsPerCta * 32, 0, s>>>(P, adj);           \
  } while (0)
#define HG_LAUNCH(NH, XM)                                                                                                \
  do {                                                                                                                   \
    if (has_ts) HG_LAUNCH2(NH, XM, true);                                                                                \
    else HG_LAUNCH2(NH, XM, false);                                                                                      \
  } while (0)
  if (nhot == 2) HG_LAUNCH(2, 0);
  else if (nhot == 3) { if (xmask & 1) HG_LAUNCH(3, 1); else HG_LAUNCH(3, 0); }
  else {
    switch (xmask & 3) {
      case 0: HG_LAUNCH(4, 0); break;
      case 1: HG_LAUNCH(4, 1); break;
      case 2: HG_LAUNCH(4, 2); break;
      default: HG_LAUNCH(4, 3);
    }
  }
#undef HG_LAUNCH
#undef HG_LAUNCH2
}

// exclusive scan of per-item record counts, two levels: every block scans 1024 items in place and publishes its sum;
// the scatter kernel adds the (<= 1024-entry) prefix of the block sums on the fly.
__global__ void __launch_bounds__(1024) item_scan_kernel(uint32_t* cnt, const uint32_t* d_nsel, uint32_t split, uint32_t* bsum) {
  __shared__ uint32_t s_w[1024 / 32 + 1];
  const uint32_t n = *d_nsel * split;
  const uint32_t i = blockIdx.x * 1024 + threadIdx.x;
  uint32_t total;
  const uint32_t ex = block_excl_scan<1024>(i < n ? cnt[i] : 0, &total, s_w);
  if (i < n) cnt[i] = ex;
  if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(256) scatter_records_kernel(const FRec* __restrict__ rec, const unsigned int* nrec, const uint32_t* __restrict__ item_off,
                                                              const uint32_t* __restrict__ bsum, uint32_t nblocks, uint32_t* d_total, uint32_t gwidth,
                                                              AggOut out, uint32_t out_cap, uint32_t rec_cap, int* err) {
  __shared__ uint32_t s_boff[1024];
  // exclusive prefix of the block sums (nblocks <= 1024), computed redundantly by every CTA
  for (uint32_t b = threadIdx.x; b < 1024; b += blockDim.x) s_boff[b] = b < nblocks ? bsum[b] : 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (uint32_t b = 0; b < nblocks; b++) { uint32_t c = s_boff[b]; s_boff[b] = run; run += c; }
    if (blockIdx.x == 0) *d_total = run;
  }
  __syncthreads();
  uint32_t n = *nrec;
  if (n > rec_cap) n = rec_cap;                     // slots reserved beyond the buffer were never written (emit() flagged 201)
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    FRec x = rec[r];
    if (x.item == 0xffffffffu) continue;          // unused tail of a warp's slot reservation
    uint32_t pos = s_boff[x.item >> 10] + item_off[x.item] + x.local;
    // the output is sized by the group bound the chunk statistics give: rows that contradict their statistics (a damaged file) can make
    // more groups than that — an error, never a write behind the arrays
    if (pos >= out_cap) { atomicExch(err, 203); continue; }
    switch (gwidth) {
      case 1: reinterpret_cast<uint8_t*>(out.gkey)[pos] = uint8_t(x.gkey); break;
      case 4: reinterpret_cast<uint32_t*>(out.gkey)[pos] = uint32_t(x.gkey); break;
      default: reinterpret_cast<uint64_t*>(out.gkey)[pos] = x.gkey;
    }
    out.bucket[pos] = x.bucket;
    out.count[pos] = x.count;
    out.sum[pos] = x.sum;
    out.min[pos] = x.mn;
    out.max[pos] = x.mx;
  }
}

__global__ void global_count_kernel(const unsigned long long* counters, AggOut out) {
  out.bucket[0] = 0;
  out.count[0] = counters[1];
  out.sum[0] = 0.0;
  out.min[0] = __longlong_as_double(0x7ff0000000000000LL);
  out.max[0] = -__longlong_as_double(0x7ff0000000000000LL);
}

struct GatePreds { int n; uint32_t kind, cls, _pad; uint32_t op[MAX_PREDS]; uint64_t lit[MAX_PREDS]; };
__global__ void __launch_bounds__(256) gate_rgs_kernel(const GateRg* __restrict__ rgs, uint32_t n, const __grid_constant__ GatePreds gp,
                                                       GateOut* __restrict__ out) {
  __shared__ uint32_t s_first, s_last, s_mask;
  for (uint32_t r = blockIdx.x; r < n; r += gridDim.x) {
    const GateRg g = rgs[r];
    const uint8_t* vals = g.vals;
    if (g.prefixed) {
      const uint32_t lv = ld32u(vals);                             // (levels of an all-valid page: a few bytes of RLE, at most a bit per row)
      vals += 4 + (lv <= g.nrows + 16u ? lv : 0u);
    }
    if (threadIdx.x == 0) { s_first = 0xffffffffu; s_last = 0; s_mask = 0; }
    __syncthreads();
    const uint32_t brows = gate_block_rows(g.nrows);
    uint32_t first = 0xffffffffu, last = 0, mask = 0;   // last = 1 + index
    for (uint32_t i = threadIdx.x; i < g.nrows; i += 256) {
      const uint64_t v = load_kind(vals, gp.kind, i);
      bool ok = true;
      for (int p = 0; p < gp.n; p++) ok = ok && op_holds(cmp_widened(v, gp.lit[p], gp.cls), gp.op[p]);
      if (ok) { first = first < i ? first : i; last = i + 1; mask |= 1u << (i / brows); }
    }
    if (last) { atomicMin(&s_first, first); atomicMax(&s_last, last); atomicOr(&s_mask, mask); }
    __syncthreads();
    if (threadIdx.x == 0) out[r] = s_last ? GateOut{s_first, s_last - 1, s_mask} : GateOut{1u, 0u, 0u};
    __syncthreads();
  }
}

}  // namespace

int gate_row_groups(hg_engine* e, const GateRg* d_rgs, uint32_t n, uint32_t type, const hg_predicate* preds, size_t np, GateOut* d_out) {
  if (n == 0) return HG_OK;
  if (np == 0 || np > size_t(MAX_PREDS)) return set_error(HG_ERR_INTERNAL, "gate_row_groups: bad predicate count");
  GatePreds gp;
  std::memset(&gp, 0, sizeof(gp));
  gp.n = int(np);
  gp.kind = kind_of(type);
  gp.cls = cmp_class(type);
  for (size_t i = 0; i < np; i++) { gp.op[i] = preds[i].op; gp.lit[i] = pred_literal(preds[i], type); }
  gate_rgs_kernel<<<int(std::min<uint32_t>(n, kNumSMs * 16u)), 256, 0, e->stream>>>(d_rgs, n, gp, d_out);
  e->launches++;
  CU_TRY(cudaGetLastError());
  return HG_OK;
}

int fused_shape(const hg_schema_desc* schema, const hg_predicate* preds, size_t np, const hg_agg_spec* agg, FusedShape* shape) {
  FusedShape& S = *shape;
  S = FusedShape{};
  S.has_group = agg->group_col >= 0;
  S.has_ts = agg->ts_col >= 0 && agg->window_ms > 0;
  S.global_mode = !S.has_group && !S.has_ts;
  if (S.has_group && agg->group_col != 0) return NOT_APPLICABLE;               // groups must be runs of the sort order
  if (S.has_ts && !(S.has_group && agg->ts_col == 1 && schema->num_primary_keys >= 2)) return NOT_APPLICABLE;
  if (S.global_mode && agg->value_col >= 0) return NOT_APPLICABLE;             // a global f64 sum is one serial chain
  if (schema->num_primary_keys < 2) return NOT_APPLICABLE;                     // the kernel keeps pk0 and pk1 in registers
  if (schema->num_primary_keys > uint32_t(MAXC)) return NOT_APPLICABLE;
  if (S.has_ts && schema->types[1] != T_I64) return NOT_APPLICABLE;
  for (int k = 0; k < 2; k++)
    if (schema->types[k] != T_U64 && schema->types[k] != T_I64) return NOT_APPLICABLE;   // pk0 / pk1 are read as 8-byte words
  // ---- column slots: PKs first, then predicate / value columns
  for (uint32_t c = 0; c < schema->num_primary_keys; c++) S.slots.push_back(c);
  auto slot_of = [&](uint32_t c) {
    for (size_t i = 0; i < S.slots.size(); i++) if (S.slots[i] == c) return int(i);
    S.slots.push_back(c);
    return int(S.slots.size() - 1);
  };
  for (size_t i = 0; i < np; i++) S.pslot[i] = slot_of(preds[i].column);
  S.value_slot = agg->value_col >= 0 ? slot_of(uint32_t(agg->value_col)) : -1;
  if (S.slots.size() > size_t(MAXC)) return NOT_APPLICABLE;
  // ---- hot slots; the predicates of one column fold into one interval of its order key:
  //   unsigned ints: key = value          signed ints: key = value ^ sign bit (of the 64-bit widened value)
  for (size_t i = 0; i < np; i++) {
    const uint32_t t = schema->types[preds[i].column];
    if (t == T_BINARY) return NOT_APPLICABLE;                                  // byte compares: the general pipeline's kernel
    if (type_is_float(t) || preds[i].op == HG_OP_NE || preds[i].op == HG_OP_IN) return NOT_APPLICABLE;    // general pipeline handles these
    if (preds[i].op == HG_OP_IN_SET) return NOT_APPLICABLE;                     // a set is no interval: the general pipeline's probe kernel
    int h = -1;
    for (int j = 0; j < S.nhot; j++) if (S.hot_slot[j] == S.pslot[i]) h = j;
    if (h < 0) {
      if (S.nhot == kHot) return NOT_APPLICABLE;                               // more than two non-PK predicate columns
      h = S.nhot++;
      S.hot_slot[h] = S.pslot[i];
    }
    S.hot_pred[h] = true;
    // literal in the key domain (64-bit widened, sign bit flipped for signed types)
    const uint64_t key = pred_literal(preds[i], t) ^ order_flip(t);
    uint64_t &lo = S.klo[h], &hi = S.khi[h];
    switch (preds[i].op) {
      case HG_OP_EQ: lo = std::max(lo, key); hi = std::min(hi, key); break;
      case HG_OP_LT: if (key == 0) S.empty_interval = true; else hi = std::min(hi, key - 1); break;
      case HG_OP_LE: hi = std::min(hi, key); break;
      case HG_OP_GT: if (key == ~0ull) S.empty_interval = true; else lo = std::max(lo, key + 1); break;
      default: lo = std::max(lo, key); break;
    }
  }
  for (int h = 0; h < kHot; h++) if (S.klo[h] > S.khi[h]) S.empty_interval = true;
  // 4-byte columns are tested in 32-bit arithmetic (make_params): an interval that misses the column type's range passes nothing
  for (int h = 2; h < S.nhot; h++) {
    const uint32_t t = schema->types[S.slots[S.hot_slot[h]]];
    if (type_width(t) == 8) continue;
    if (type_is_signed(t) ? (S.khi[h] < kI32KeyLo || S.klo[h] > kI32KeyHi) : S.klo[h] > 0xffffffffull) S.empty_interval = true;
  }
  // the LAST hot column is the gate of the late-materialising kernel: put the narrower of two extra columns there
  if (S.nhot == 4 && type_width(schema->types[S.slots[S.hot_slot[2]]]) < type_width(schema->types[S.slots[S.hot_slot[3]]])) {
    std::swap(S.hot_slot[2], S.hot_slot[3]);
    std::swap(S.klo[2], S.klo[3]);
    std::swap(S.khi[2], S.khi[3]);
  }
  return HG_OK;
}

namespace {

// The fused scan's counter block: zeroed by one memset before the first launch, read back by one D2H copy after the last.
// FParams::work points at its start.  The work counters, the row counters and the error word each start a 64-byte line.
struct WorkBlock {
  uint32_t item_ticket;            // fused_scan_kernel: next work item (FParams::work[0])
  uint32_t rec_slots;              // fused_scan_kernel: record slots reserved (FParams::work[1]); scatter_records_kernel reads it
  uint32_t groups;                 // scatter_records_kernel: groups written
  uint32_t nsel;                   // select_rgs_kernel, then compact_sel_kernel: selected row groups (FParams::d_nsel)
  uint32_t gate_fallback;           // k::snappy_gate_pages: gate chunks decompressed because the bit path declined a page (trace)
  uint32_t _pad0[11];
  unsigned long long counters[4];  // FParams::counters: select_rgs_kernel writes [2], fused_scan_kernel [0], [1] and [3]
  uint64_t _pad1[4];
  int err;                         // FParams::err, SnappyJob::err: a device error code (201-203: damaged data) from any kernel of the call
  uint32_t _pad2;
  unsigned int snappy_ticket[2];   // SnappyJob::ticket of the gate column's job and of the other columns' job
};
static_assert(offsetof(WorkBlock, item_ticket) == 0 && offsetof(WorkBlock, rec_slots) == 4, "FParams::work indexes the block");
static_assert(offsetof(WorkBlock, counters) == 64 && offsetof(WorkBlock, err) == 128 && sizeof(WorkBlock) <= 256,
              "own 64-byte lines; hg_engine::h_small holds 256 bytes");

// One fused aggregate call, planned and launched in stages (try_scan_aggregate calls them in order)
struct FusedPlan {
  hg_engine* e;
  const hg_schema_desc* schema;
  const hg_predicate* preds;
  size_t np;
  const hg_agg_spec* agg;
  AggBuffers* out;
  FusedShape S;
  HostClock::time_point t0, t1, t2;
  // plan_files
  std::vector<SstResident*> files;        // in pk0 order
  uint64_t rows_in_files = 0;
  uint32_t total_rgs = 0;
  // lay_out_scratch
  bool slot_snappy[MAXC] = {false};
  uint64_t slot_comp[MAXC] = {0};
  uint64_t scratch_stride = 0, scratch_per_rg = 0;
  bool value_stored = false;
  int region[MAXC];
  int nregions = 0;
  // size_groups
  uint64_t bound = 1, rec_cap = 0;
  uint32_t split = 1, nitems = 0;
  // alloc: destroyed in reverse order of declaration, and the arena takes back only its most recent allocation
  DevBuf d_ssts, d_files, d_sel, d_sel2, d_rec, d_item, d_work, d_adj, d_keep, d_bsum, d_bases, d_vseg, d_gflags, d_scratch, d_lpt;
  WorkBlock* work = nullptr;
  // make_params
  FParams P;
  bool gated = false, gate_first = false;
  int xmask = 0;

  bool need_snappy() const { return nregions > 0; }
  int gate_slot() const { return S.hot_slot[S.nhot - 1]; }
  int plan_files(const hg_sst_desc* ssts, size_t n);
  int empty_answer();
  void lay_out_scratch();
  int size_groups();
  int alloc();
  int make_params();
  void set_hot_params();
  k::SnappyJob make_job(const std::vector<int>& job_slots, unsigned int* ticket) const;
  void decompress(const Launch& L);
  int launch();
  int read_back();
};

// residency, the per-file preconditions, PK-disjointness and the stream order of the files (row groups are pruned and listed on the device)
int FusedPlan::plan_files(const hg_sst_desc* ssts, size_t n) {
  for (size_t i = 0; i < n; i++) {
    auto it = e->ssts.find(ssts[i].id);
    if (it == e->ssts.end()) return set_error(HG_ERR_INTERNAL, "sst not resident after load");
    SstResident* f = it->second.get();
    rows_in_files += f->rows_total;
    if (f->rows_total == 0) continue;
    for (uint32_t c : S.slots)
      if (!f->row_addressable(c)) return NOT_APPLICABLE;
    if (!S.global_mode && (!f->col_has_minmax[0] || (S.has_ts && !f->col_has_minmax[1]))) return NOT_APPLICABLE;
    files.push_back(f);
  }
  if (files.size() > 1) {
    std::vector<Pk0Range> ranges;
    std::vector<size_t> order;
    for (SstResident* f : files) ranges.push_back(f->pk0);
    if (!pk0_disjoint(ranges, schema->types[0], &order)) return NOT_APPLICABLE;   // not provably PK-disjoint
    const std::vector<SstResident*> given = files;
    for (size_t j = 0; j < order.size(); j++) files[j] = given[order[j]];
  }
  for (SstResident* f : files) total_rgs += uint32_t(f->rg_rows.size());
  return HG_OK;
}

// a contradictory conjunction (an empty time range, `= a AND = b`, `< min`) passes no row: the answer is known without a launch, and it
// is the general pipeline's for zero surviving rows — no group, the global count(*) included
int FusedPlan::empty_answer() {
  CU_TRY(out->alloc(0, e->stream));
  out->G = 0;
  e->stats.rows_in_files = rows_in_files;
  e->stats.path = 1;
  return HG_OK;
}

// Snappy pages (WriteConfig::default, config.rs:120-133) are decompressed into per-(row group, slot) scratch regions before the scan
// kernel runs.  The value column's stored (literal-only) Snappy pages are read in place through a per-row-group segment table (VSeg); its
// other pages — a random f64 column still yields the odd page with a copy element — are decompressed like any column and the table
// points at the scratch.  value_stored = that table is in use; value_all_stored = no page of the column needs scratch at all.
void FusedPlan::lay_out_scratch() {
  bool value_all_stored = true;
  for (size_t i = 0; i < S.slots.size(); i++)
    for (SstResident* f : files) {
      const uint32_t c = S.slots[i];
      if (f->col_any_snappy[c]) { slot_snappy[i] = true; scratch_stride = std::max<uint64_t>(scratch_stride, f->col_max_scratch[c]); }
      slot_comp[i] += f->col_comp_bytes[c];
      if (int(i) == S.value_slot) {
        if (f->col_snappy_any_stored[c]) value_stored = true;
        if (f->col_any_snappy[c] && !f->col_snappy_all_stored[c]) value_all_stored = false;
      }
    }
  if (S.value_slot >= 0) {
    if (!slot_snappy[S.value_slot]) value_stored = false;
    for (int h = 0; h < S.nhot; h++) if (S.hot_slot[h] == S.value_slot) value_stored = false;   // hot columns are addressed contiguously
    for (int k2 = 0; k2 < int(schema->num_primary_keys); k2++) if (k2 == S.value_slot) value_stored = false;
  }
  scratch_stride = (scratch_stride + 255) & ~uint64_t(255);
  // the gate column's bitmaps follow a row group's regions: one bit per row of the largest row group
  uint32_t max_rg_rows = 0;
  for (SstResident* f : files)
    for (uint32_t r : f->rg_rows) max_rg_rows = std::max(max_rg_rows, r);
  const uint64_t bits_bytes = (uint64_t((max_rg_rows + 31) / 32) * 4 + 255) & ~uint64_t(255);
  for (size_t i = 0; i < S.slots.size(); i++)
    region[i] = (slot_snappy[i] && !(value_stored && value_all_stored && int(i) == S.value_slot)) ? nregions++ : -1;
  scratch_per_rg = uint64_t(nregions) * scratch_stride + bits_bytes;
}

// upper bound on the number of groups from chunk statistics (sizes the unordered record buffer), and the work items
int FusedPlan::size_groups() {
  if (!S.global_mode) {
    if (type_is_float(schema->types[0])) return NOT_APPLICABLE;
    bound = 0;
    if (!S.has_ts) {
      for (SstResident* f : files) bound += f->group_bound;
    } else {
      for (SstResident* f : files) {
        const size_t ncols = size_t(f->meta.ncols);
        for (size_t g = 0; g < f->rg_rows.size(); g++) {
          const RgCol* rc = &f->rgcol[g * ncols];
          const uint64_t rows = f->rg_rows[g];
          uint64_t span = rc[0].mx - rc[0].mn + 1;
          // buckets per pk0 value: the ts distance mx - mn as u64 (no signed overflow across the i64 range), saturated
          uint64_t per = std::min<uint64_t>((rc[1].mx - rc[1].mn) / uint64_t(agg->window_ms), 1ull << 33) + 2;
          uint64_t gcount = (span == 0 || span > (1ull << 32) || per > (1ull << 32)) ? rows : span * per;
          bound += std::min<uint64_t>(gcount, rows) + 1;
        }
      }
    }
    // more than ~1 group per warp-slice: the per-survivor walk dominates and the materialising pipeline (thread per
    // group) is faster
    if (bound > rows_in_files / 32 + 1024) return NOT_APPLICABLE;
  }
  if (bound >= 0xfffffff0ull || rows_in_files >= 0xfffffff0ull) return NOT_APPLICABLE;
  // split row groups into enough work items for ~4 items per resident warp (dynamic ticket => good balance);
  // boundaries are then aligned to key-run starts by item_bounds_kernel
  constexpr uint64_t kItemsPerWarp = 4;
  while (split < 8 && uint64_t(total_rgs) * split < uint64_t(kNumSMs) * 32 * kItemsPerWarp) split *= 2;
  nitems = total_rgs * split;      // upper bound: pruning only removes items
  if ((uint64_t(nitems) + 1023) / 1024 > 1024) return NOT_APPLICABLE;   // two-level item scan covers 1 M work items
  rec_cap = bound + uint64_t(kNumSMs) * 8 * kWarpsPerCta * 32;          // + one partly used 32-slot reservation per warp
  return HG_OK;
}

int FusedPlan::alloc() {
  cudaStream_t s = e->stream;
  CU_TRY(d_work.alloc(sizeof(WorkBlock), s));
  CU_TRY(cudaMemsetAsync(d_work.p, 0, sizeof(WorkBlock), s));
  work = d_work.as<WorkBlock>();
  CU_TRY(d_rec.alloc(size_t(rec_cap) * sizeof(FRec) + 64, s));
  CU_TRY(d_item.alloc(size_t(nitems + 1) * sizeof(uint32_t) + 64, s));
  CU_TRY(d_adj.alloc(size_t(nitems + 2) * sizeof(uint64_t), s));
  CU_TRY(d_sel.alloc(size_t(total_rgs + 1) * sizeof(RgSel), s));
  CU_TRY(d_keep.alloc(size_t(total_rgs + 1) * sizeof(uint32_t), s));
  CU_TRY(d_bsum.alloc(1024 * sizeof(uint32_t), s));
  CU_TRY(d_bases.alloc(size_t(total_rgs + 1) * MAXC * sizeof(uint8_t*), s));
  if (value_stored) CU_TRY(d_vseg.alloc(size_t(total_rgs + 1) * sizeof(VSeg), s));
  if (need_snappy()) {
    CU_TRY(d_sel2.alloc(size_t(total_rgs + 1) * sizeof(RgSel), s));
    CU_TRY(d_gflags.alloc(size_t(total_rgs) + 16, s));
    CU_TRY(d_lpt.alloc(size_t(total_rgs + 1) * sizeof(uint32_t), s));
    CU_TRY(d_scratch.alloc(size_t(total_rgs) * size_t(scratch_per_rg) + 256, s));
  }
  CU_TRY(out->alloc(bound, s));
  return HG_OK;
}

// uploads the file tables and fills the kernels' parameter block
int FusedPlan::make_params() {
  std::vector<SstDev> sd(files.size());
  std::vector<FileDev> fdv(files.size());
  uint32_t rgb = 0;
  for (size_t i = 0; i < files.size(); i++) {
    SstResident* f = files[i];
    sd[i] = SstDev{f->d_bytes, f->d_pages, f->d_chunks, uint32_t(f->meta.ncols), uint32_t(f->meta.rgs.size())};
    fdv[i] = FileDev{f->d_rgcol, f->d_rg_rows, rgb, uint32_t(f->rg_rows.size()), uint32_t(f->meta.ncols), 0, f->d_bytes};
    rgb += uint32_t(f->rg_rows.size());
  }
  CU_TRY(d_ssts.alloc(sd.size() * sizeof(SstDev), e->stream));
  CU_TRY(d_files.alloc(fdv.size() * sizeof(FileDev), e->stream));
  int urc = stage_upload(e, d_ssts.p, sd.data(), sd.size() * sizeof(SstDev));
  if (!urc) urc = stage_upload(e, d_files.p, fdv.data(), fdv.size() * sizeof(FileDev));
  if (urc) return urc;

  std::memset(&P, 0, sizeof(P));
  P.ssts = d_ssts.as<SstDev>();
  P.sel = d_sel.as<RgSel>();
  P.d_nsel = &work->nsel;
  P.bases = d_bases.as<const uint8_t*>();
  P.split = split;
  P.nslots = int(S.slots.size());
  for (size_t i = 0; i < S.slots.size(); i++) {
    uint32_t t = schema->types[S.slots[i]];
    P.col[i] = S.slots[i];
    P.kind[i] = kind_of(t);
    P.cls[i] = cmp_class(t);
  }
  P.npk = int(schema->num_primary_keys);
  P.has_group = S.has_group;
  P.has_ts = S.has_ts;
  P.value_slot = S.value_slot;
  P.global_mode = S.global_mode;
  set_hot_params();
  P.npred = int(np);
  for (size_t i = 0; i < np; i++) {
    const uint32_t t = schema->types[preds[i].column];
    P.pslot[i] = S.pslot[i];
    P.pop[i] = preds[i].op;
    P.plit[i] = pred_literal(preds[i], t);
    P.pcol[i] = preds[i].column;
    P.pcls[i] = cmp_class(t);
    P.pbloom[i] = preds[i].op == HG_OP_EQ && bloom_literal_hash(P.plit[i], t, &P.phash[i]) ? 1u : 0u;
  }
  P.window_ms = S.has_ts ? agg->window_ms : 1;
  P.scratch = d_scratch.as<uint8_t>();
  P.scratch_stride = scratch_stride;
  for (int i = 0; i < MAXC; i++) P.region[i] = i < int(S.slots.size()) ? region[i] : -1;
  P.value_stored = value_stored ? 1 : 0;
  P.vseg = d_vseg.as<VSeg>();
  P.rec = d_rec.as<FRec>();
  P.rec_cap = uint32_t(rec_cap);
  P.item_cnt = d_item.as<uint32_t>();
  P.work = &work->item_ticket;
  P.counters = work->counters;
  P.err = &work->err;
  // late materialisation needs a real interval test on the last hot column (the gate); gate-first decompression (launch) lets
  // gate_rg_kernel keep one bit per row of the gate column for the gated kernel's sweeps
  gated = !(e->flags & HG_FLAG_NO_LATE_MATERIALIZATION) && P.hot_haspred[S.nhot - 1] != 0;
  gate_first = need_snappy() && gated && region[gate_slot()] >= 0;
  P.gate_bits = gate_first ? 1 : 0;
  // a 4-byte gate column that is neither a key nor the value column is only ever tested: its row-group gate can work from the compressed
  // pages (k::snappy_gate_pages) without decompressing the column at all.  That path's work is per Snappy element and it hands a page
  // of more than snp::kGateCap table entries back to the byte decoder, so it is taken for run-coded columns only: under half a
  // compressed byte per row (the bench's tag: 0.19; a tag that changes every few rows: 1.4-1.6, and every page would go back)
  const int gs = gate_slot();
  const bool runs = slot_comp[gs] * 2 < rows_in_files;
  P.gate_slot = gate_first && runs && P.kind[gs] != K_RAW64 && gs >= P.npk && gs != S.value_slot ? gs : -1;
  P.bits_off = uint64_t(nregions) * scratch_stride;
  return HG_OK;
}

// the hot slots' interval tests, and xmask: bit h - 2 set = extra hot column h is 4 bytes wide
void FusedPlan::set_hot_params() {
  for (int h = 0; h < kHot; h++) {
    const int sl = h < S.nhot ? S.hot_slot[h] : 0;
    const uint32_t t = schema->types[S.slots[sl]];
    const bool w8 = (t == T_U64 || t == T_I64 || t == T_F64);
    P.hot_slot[h] = sl;
    P.hot_haspred[h] = (h < S.nhot && (S.klo[h] != 0 || S.khi[h] != ~0ull)) ? 1 : 0;
    // 8-byte columns: key = raw ^ signflip.  4-byte columns are tested in 32-bit arithmetic: the widened key of a signed
    // value v is sext(v) ^ 2^63, ordered like (v ^ 2^31) as unsigned 32-bit; rebase the interval into that domain.
    // (an interval outside the 32-bit range was found empty by fused_shape)
    uint64_t lo = S.klo[h], hi = S.khi[h];
    if (w8) P.hot_flip[h] = order_flip(t);
    else if (type_is_signed(t)) {
      P.hot_flip[h] = 1ull << 31;
      lo = lo < kI32KeyLo ? 0 : lo - kI32KeyLo;
      hi = hi > kI32KeyHi ? 0xffffffffull : hi - kI32KeyLo;
    } else {
      P.hot_flip[h] = 0;
      hi = std::min<uint64_t>(hi, 0xffffffffull);
    }
    P.hot_lo[h] = lo;
    P.hot_span[h] = hi >= lo ? hi - lo : 0;
    if (h >= 2 && h < S.nhot && !w8) xmask |= 1 << (h - 2);
  }
}

// a decompression job over the given slots, in descending order of compressed bytes (long pages first, short ones fill the tail)
k::SnappyJob FusedPlan::make_job(const std::vector<int>& job_slots, unsigned int* ticket) const {
  k::SnappyJob J;
  std::memset(&J, 0, sizeof(J));
  J.ssts = P.ssts; J.sel = P.sel; J.d_nsel = P.d_nsel; J.nsel = 0; J.ncols = int(job_slots.size());
  std::vector<int> ord(job_slots.size());
  for (size_t i = 0; i < ord.size(); i++) ord[i] = int(i);
  std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return slot_comp[job_slots[a]] > slot_comp[job_slots[b]]; });
  for (size_t i = 0; i < job_slots.size(); i++) {
    J.col[i] = S.slots[job_slots[i]];
    J.region[i] = uint32_t(region[job_slots[i]]);
    J.order[i] = uint8_t(ord[i]);
    J.skip_stored[i] = (value_stored && job_slots[i] == S.value_slot) ? 1 : 0;   // stored pages of the value column stay where they are
  }
  J.fixed_stride = scratch_stride; J.scratch = d_scratch.as<uint8_t>(); J.ticket = ticket; J.err = P.err;
  return J;
}

// Snappy slots into their scratch regions.  Gate first: decompress the gate column, find the row groups with a passing row (and keep
// one bit per row of the column), drop the others, decompress the rest for the others.
void FusedPlan::decompress(const Launch& L) {
  cudaStream_t s = e->stream;
  const int gs = gate_slot();
  std::vector<int> first, rest;
  for (int i = 0; i < int(S.slots.size()); i++) {
    if (region[i] < 0) continue;
    if (gate_first && i == gs) first.push_back(i); else rest.push_back(i);
  }
  if (!first.empty()) {
    const uint32_t gt = schema->types[S.slots[gs]];
    const bool w4 = !(gt == T_U64 || gt == T_I64 || gt == T_F64);
    const int h = S.nhot - 1;
    if (P.gate_slot >= 0) {
      // straight from the compressed pages: one bit per row, the column itself is not written
      k::GateJob G;
      G.J = make_job(first, &work->snappy_ticket[0]);
      G.sel = d_sel.as<RgSel>(); G.bits_off = P.bits_off;
      G.flip = uint32_t(P.hot_flip[h]); G.lo = uint32_t(P.hot_lo[h]); G.span = uint32_t(P.hot_span[h]);
      G.flags = d_gflags.as<uint8_t>(); G.fallback = &work->gate_fallback;
      k::snappy_gate_pages(L, G, total_rgs);
    } else {
      k::snappy_pages(L, make_job(first, &work->snappy_ticket[0]), total_rgs);
      if (w4) gate_rg_kernel<true><<<kNumSMs * 8, 256, 0, s>>>(P, d_sel.as<RgSel>(), gs, P.hot_flip[h], P.hot_lo[h], P.hot_span[h], d_gflags.as<uint8_t>());
      else gate_rg_kernel<false><<<kNumSMs * 8, 256, 0, s>>>(P, d_sel.as<RgSel>(), gs, P.hot_flip[h], P.hot_lo[h], P.hot_span[h], d_gflags.as<uint8_t>());
      L.tick();
    }
    compact_sel_kernel<<<1, 1024, 0, s>>>(d_sel.as<RgSel>(), d_gflags.as<uint8_t>(), &work->nsel, d_sel2.as<RgSel>(), d_lpt.as<uint32_t>());
    L.tick();
    P.sel = d_sel2.as<RgSel>();
  }
  if (!rest.empty()) {
    k::SnappyJob J2 = make_job(rest, &work->snappy_ticket[1]);
    // after the row-group gate only the rows up to the last gate-passing row (+1) of a row group are ever read from the
    // non-gate columns — except pk0, which the work-item boundaries probe anywhere (and pk1 when groups are time buckets)
    if (!first.empty() && !S.has_ts)
      for (size_t i = 0; i < rest.size(); i++) J2.partial[i] = rest[i] != 0 ? 1 : 0;
    if (!first.empty()) { J2.sel = P.sel; J2.lpt = d_lpt.as<uint32_t>(); }       // longest pages first (compact_sel_kernel)
    k::snappy_pages(L, J2, total_rgs * uint32_t(rest.size()));
  }
}

// prune -> select -> decompress -> slot bases -> item bounds -> fused scan -> records in stream order (or the global count)
int FusedPlan::launch() {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const FileDev* fd = d_files.as<FileDev>();
  prune_rgs_kernel<<<(total_rgs + 255) / 256, 256, 0, s>>>(P, fd, int(files.size()), total_rgs,
                                                           (e->flags & HG_FLAG_NO_PRUNING) ? 0 : ((e->flags & HG_FLAG_NO_BLOOM_FILTER) ? 1 : 3),
                                                           d_keep.as<uint32_t>());
  L.tick();
  CU_TRY(cudaFuncSetAttribute(select_rgs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));   // per device
  const uint32_t smem_words = size_t(total_rgs) * 4 <= 200 * 1024 ? total_rgs : 0;
  select_rgs_kernel<<<1, 1024, size_t(smem_words) * 4, s>>>(fd, int(files.size()), total_rgs, d_keep.as<uint32_t>(), d_sel.as<RgSel>(),
                                                            &work->nsel, work->counters, smem_words, scratch_per_rg);
  L.tick();
  CU_TRY(cudaEventRecord(e->evd0, s));
  if (need_snappy()) decompress(L);
  CU_TRY(cudaEventRecord(e->evd1, s));
  slot_bases_kernel<<<(total_rgs * MAXC + 255) / 256, 256, 0, s>>>(P, d_bases.as<const uint8_t*>());
  L.tick();
  const uint32_t nb = (nitems + 1 + kBoundsPerWarp - 1) / kBoundsPerWarp;      // warps
  const int bctas = int((uint64_t(nb) * 32 + 255) / 256);
  if (S.has_ts) item_bounds_kernel<true><<<bctas, 256, 0, s>>>(P, d_adj.as<uint64_t>());
  else item_bounds_kernel<false><<<bctas, 256, 0, s>>>(P, d_adj.as<uint64_t>());
  L.tick();
  CU_TRY(cudaEventRecord(e->evk0, s));
  // 2 slices per block, 4 CTAs/SM, L2 prefetch 2 blocks / sweeps ahead
  const int ctas = int(std::min<uint64_t>((uint64_t(nitems) + kWarpsPerCta - 1) / kWarpsPerCta, uint64_t(kNumSMs) * 8));
  launch_fused<2, 4>(S.nhot, xmask, S.has_ts, gated, ctas, s, P, d_adj.as<uint64_t>());
  L.tick();
  CU_TRY(cudaEventRecord(e->evk1, s));
  if (S.global_mode) {
    global_count_kernel<<<1, 1, 0, s>>>(work->counters, out->out());
    L.tick();
  } else {
    const uint32_t sblocks = (nitems + 1023) / 1024;
    item_scan_kernel<<<sblocks, 1024, 0, s>>>(d_item.as<uint32_t>(), &work->nsel, split, d_bsum.as<uint32_t>());
    L.tick();
    scatter_records_kernel<<<kNumSMs * 4, 256, 0, s>>>(d_rec.as<FRec>(), &work->rec_slots, d_item.as<uint32_t>(), d_bsum.as<uint32_t>(), sblocks,
                                                       &work->groups, out->gwidth, out->out(), uint32_t(std::min<uint64_t>(bound, 0xffffffffu)),
                                                       uint32_t(std::min<uint64_t>(rec_cap, 0xffffffffu)), &work->err);
    L.tick();
  }
  return HG_OK;
}

// one D2H copy of the counter block, the device error, the stats
int FusedPlan::read_back() {
  WorkBlock w;
  std::memset(&w, 0, sizeof(w));
  if (total_rgs > 0) {
    const auto t3 = HostClock::now();
    if (!e->h_small) CU_TRY(cudaMallocHost(&e->h_small, 256));
    CU_TRY(cudaMemcpyAsync(e->h_small, work, sizeof(WorkBlock), cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    std::memcpy(&w, e->h_small, sizeof(w));
    const auto t4 = HostClock::now();
    if (trace_on())
      fprintf(stderr, "[fused] plan %.0f us, bound+alloc %.0f us, upload+launch %.0f us, wait %.0f us (row groups %u, max items %u, gate chunks decompressed %u)\n",
              elapsed_us(t0, t1), elapsed_us(t1, t2), elapsed_us(t2, t3), elapsed_us(t3, t4), total_rgs, nitems, w.gate_fallback);
    if (w.err >= 201 && w.err <= 203)
      return set_error(HG_ERR_FORMAT, "fused scan: rows contradict their chunk statistics or a page is damaged (device error " + std::to_string(w.err) + ")");
    if (w.err) return set_error(HG_ERR_INTERNAL, "fused scan: device error " + std::to_string(w.err));
    float kms = 0;
    cudaEventElapsedTime(&kms, e->evk0, e->evk1);
    e->stats.kernel_ms = kms;
    if (need_snappy()) { cudaEventElapsedTime(&kms, e->evd0, e->evd1); e->stats.decomp_ms = kms; }
  }
  out->G = S.global_mode ? (w.counters[1] > 0 ? 1u : 0u) : w.groups;   // like GROUP BY: no surviving rows, no group
  e->stats.rows_in_files = rows_in_files;
  e->stats.rows_decoded = w.counters[2];
  e->stats.rows_materialized = w.counters[3];
  e->stats.rows_filtered = w.counters[0];
  e->stats.rows_out = w.counters[1];
  e->stats.groups_out = out->G;
  e->stats.path = 1;
  return HG_OK;
}

}  // namespace

int try_scan_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n, const hg_predicate* preds,
                       size_t np, const hg_agg_spec* agg, AggBuffers* out) {
  FusedPlan F{e, schema, preds, np, agg, out};
  if (fused_shape(schema, preds, np, agg, &F.S) == NOT_APPLICABLE) return NOT_APPLICABLE;
  F.t0 = HostClock::now();
  int rc = F.plan_files(ssts, n);
  if (rc) return rc;
  out->gtype = F.S.has_group ? schema->types[0] : uint32_t(T_U64);
  out->gwidth = F.S.has_group ? type_width(out->gtype) : 8;
  if (F.S.empty_interval) return F.empty_answer();
  F.lay_out_scratch();
  F.t1 = HostClock::now();
  if ((rc = F.size_groups()) || (rc = F.alloc())) return rc;
  F.t2 = HostClock::now();
  if (F.total_rgs > 0 && ((rc = F.make_params()) || (rc = F.launch()))) return rc;
  return F.read_back();
}


}  // namespace fused
}  // namespace horae
