// sst_writer.cu — GPU Parquet page encoder + SST assembly: the second half of Executor::do_compaction
// (compaction/executor.rs:173-203: AsyncArrowWriter over the merged stream) and of write_batch (storage.rs:189-225), with
// the writer properties of build_write_props (storage.rs:258-298) and WriteConfig::default (config.rs:120-133):
// row groups of max_row_group_size rows, one DataPage V1 per column chunk, RLE/bit-packed definition levels (every field is
// nullable), chunk statistics (min / max / null_count), sorting_columns = primary keys ascending nulls first, Thrift-compact footer.
// Per column (hg_write_props.columns, config.rs:54-133): PLAIN or DELTA_BINARY_PACKED values, optionally a dictionary (PLAIN dictionary
// page + RLE_DICTIONARY data page), uncompressed, Snappy or Zstd pages (config.rs:78-94), optionally a split-block bloom filter per chunk
// (enable_bloom_filter, config.rs:100 / 113), placed after its row group's chunks like parquet-rs's BloomFilterPosition::AfterRowGroup.
//
// Device work: page bodies (level prefix + compacted non-null values), chunk statistics, bloom filters, DELTA / dictionary encoding, page
// compression and the final gather into one contiguous file image.  Host work: the few KB of Thrift (page headers, footer) and the offsets.
//
// The Snappy compressor is written for what these pages hold — fixed-width numbers: value i is compared with value i-1
// (8-byte columns: how many HIGH bytes agree; 4-byte columns: equal or not) and the page becomes literal runs, 2-byte
// copies of the agreeing high bytes (offset = value width) and 64-byte run-length copies.  Every value computes its own
// emitted size, one prefix sum gives all positions, every value writes its own bytes: no serial parse, any Snappy decoder
// reads the result.  (On the synthetic metric data it lands within a few percent of the reference compressor's ratio.)
//
// The Zstandard compressor (RFC 8878) finds its matches the same way, plus one far candidate per value (the most recent earlier equal
// value of the page, from a hash table in shared memory), and writes one frame per page: raw literals, sequences coded with the
// predefined or RLE FSE tables, raw / RLE / compressed blocks, whichever is smallest.  See zstd_encode_kernel.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstring>
#include <string>
#include <vector>

#include "block_scan.h"
#include "engine_internal.h"
#include "sst_writer.h"

#define SNP_FN __device__ __forceinline__
#define SNP_CONST __constant__ const
#include "zstd_tables.h"
#include "bloom.h"

namespace horae {
namespace writer {

namespace {

constexpr int kThreads = 256;

struct PageMetaDev {
  uint32_t uncomp_size, comp_size, null_count, has_minmax;
  uint64_t mn, mx;             // PLAIN bytes of min / max (little endian, low `width` bytes)
  uint32_t head;               // bytes the compressors copy as one literal head before the values / 4-byte words (the level prefix)
  uint32_t enc;                // data page encoding: ENC_PLAIN, ENC_DELTA_BINARY_PACKED or ENC_RLE_DICT
  uint32_t ndict, _pad;        // RLE_DICTIONARY: entries of the chunk's dictionary page
};

struct PageJob {
  const void* vals;            // dense column
  const uint8_t* valid;        // one byte per row or nullptr
  uint32_t type, width;        // hg_type, value width in the column array
  uint32_t pwidth;             // physical width in the page (4 or 8)
  uint32_t encoding;           // ENC_PLAIN or ENC_DELTA_BINARY_PACKED (the fallback when a dictionary is refused)
  uint32_t dictionary;         // 1: try a dictionary page
};

// One page for a compressor: its bytes are [head][whole values of `w` bytes] (head = meta[meta].head, the rest of the page is a multiple of w)
struct CompUnit {
  const uint8_t* in;
  uint8_t* out;
  uint32_t meta, w;
};

// ULEB128 varints of u32 or u64 values (the type is the caller's: the loop runs at its width)
template <typename T>
__device__ __forceinline__ uint32_t varint_put(uint8_t* p, T v) {
  uint32_t n = 0;
  while (v >= 0x80) { p[n++] = uint8_t(v | 0x80); v >>= 7; }
  p[n++] = uint8_t(v);
  return n;
}
template <typename T>
__device__ __forceinline__ uint32_t varint_len(T v) { uint32_t n = 0; while (v >= 0x80) { n++; v >>= 7; } return n + 1; }

// rows of row group g of R rows cut into groups of rg_rows
__host__ __device__ __forceinline__ uint32_t rows_of_rg(uint32_t g, uint32_t R, uint32_t rg_rows) {
  return (R - g * rg_rows) < rg_rows ? (R - g * rg_rows) : rg_rows;
}

__device__ __forceinline__ uint64_t load_phys(const PageJob& j, uint32_t row) {
  // the value as PLAIN physical bytes: 1/2-byte integers widen to INT32 (sign- or zero-extended by their type)
  switch (j.type) {
    case T_U8: return reinterpret_cast<const uint8_t*>(j.vals)[row];
    case T_I8: return uint32_t(int32_t(reinterpret_cast<const int8_t*>(j.vals)[row]));
    case T_U16: return reinterpret_cast<const uint16_t*>(j.vals)[row];
    case T_I16: return uint32_t(int32_t(reinterpret_cast<const int16_t*>(j.vals)[row]));
    case T_U32: case T_I32: case T_F32: return reinterpret_cast<const uint32_t*>(j.vals)[row];
    default: return reinterpret_cast<const uint64_t*>(j.vals)[row];
  }
}

// One block per page (row group g, column c): [u32 level bytes][definition levels][PLAIN values of the non-null rows].  A page body of
// m rows takes at most page_body_bytes(m).
__host__ __device__ __forceinline__ uint64_t align64(uint64_t x) { return (x + 63) & ~uint64_t(63); }
__host__ __device__ __forceinline__ uint64_t page_body_bytes(uint32_t m) { return align64(uint64_t(16) + (m + 7) / 8 + 8 + uint64_t(m) * 8); }
__global__ void __launch_bounds__(kThreads) page_body_kernel(const PageJob* __restrict__ jobs, uint32_t ncols, uint32_t R, uint32_t rg_rows,
                                                            uint8_t* __restrict__ body, uint64_t bstride, PageMetaDev* __restrict__ meta) {
  __shared__ uint32_t s_w[9];
  __shared__ uint32_t s_nulls, s_prefix;
  __shared__ unsigned long long s_mn, s_mx;
  __shared__ uint32_t s_seen;
  const uint32_t page = blockIdx.x, g = page / ncols, c = page % ncols;
  const PageJob j = jobs[c];
  const uint32_t row0 = g * rg_rows, rows = rows_of_rg(g, R, rg_rows);
  uint8_t* out = body + uint64_t(page) * bstride;
  const int tid = threadIdx.x;
  if (tid == 0) { s_nulls = 0; s_mn = ~0ull; s_mx = 0; s_seen = 0; }
  __syncthreads();
  // ---- null count
  uint32_t nulls = 0;
  if (j.valid) for (uint32_t i = tid; i < rows; i += kThreads) nulls += j.valid[row0 + i] == 0;
  for (int d = 16; d > 0; d >>= 1) nulls += __shfl_down_sync(0xffffffffu, nulls, d);
  if ((tid & 31) == 0 && nulls) atomicAdd(&s_nulls, nulls);
  __syncthreads();
  const uint32_t nnull = s_nulls;
  // ---- definition levels (bit width 1): one RLE run when uniform, else one bit-packed run of ceil(rows/8) groups
  if (tid == 0) {
    uint32_t n = 0;
    uint8_t* lv = out + 4;
    if (nnull == 0 || nnull == rows) { n = varint_put(lv, rows << 1); lv[n++] = nnull == 0 ? 1 : 0; }
    else { const uint32_t groups = (rows + 7) / 8; n = varint_put(lv, (groups << 1) | 1u); n += groups; }
    out[0] = uint8_t(n); out[1] = uint8_t(n >> 8); out[2] = uint8_t(n >> 16); out[3] = uint8_t(n >> 24);
    s_prefix = 4 + n;
  }
  __syncthreads();
  const uint32_t prefix = s_prefix;
  if (nnull != 0 && nnull != rows) {
    const uint32_t groups = (rows + 7) / 8;
    uint8_t* bits = out + prefix - groups;
    for (uint32_t b = tid; b < groups; b += kThreads) {
      uint32_t v = 0;
#pragma unroll
      for (int k2 = 0; k2 < 8; k2++) { const uint32_t i = b * 8 + k2; if (i < rows && j.valid[row0 + i]) v |= 1u << k2; }
      bits[b] = uint8_t(v);
    }
  }
  // ---- values of the non-null rows, compacted in order; statistics
  uint8_t* vout = out + prefix;
  uint32_t running = 0;
  unsigned long long mn = ~0ull, mx = 0;
  bool seen = false;
  for (uint32_t base = 0; base < rows; base += kThreads) {
    const uint32_t i = base + tid;
    const uint32_t v = (i < rows && (!j.valid || j.valid[row0 + i])) ? 1u : 0u;
    uint32_t total;
    const uint32_t k2 = running + block_excl_scan<kThreads>(v, &total, s_w);
    if (v) {
      const uint64_t x = load_phys(j, row0 + i);
      // (the page body starts 64-byte aligned; the level prefix is usually 8 bytes, so the values are naturally aligned)
      if (j.pwidth == 8) {
        uint8_t* q = vout + size_t(k2) * 8;
        if ((prefix & 7) == 0) *reinterpret_cast<uint64_t*>(q) = x;
        else for (int b = 0; b < 8; b++) q[b] = uint8_t(x >> (8 * b));
      } else {
        uint8_t* q = vout + size_t(k2) * 4;
        if ((prefix & 3) == 0) *reinterpret_cast<uint32_t*>(q) = uint32_t(x);
        else for (int b = 0; b < 4; b++) q[b] = uint8_t(x >> (8 * b));
      }
      const uint64_t xw = widen(x, j.type);
      if (!widened_is_nan(xw, j.type)) {
        const uint64_t key = order_key(xw, j.type);
        mn = key < mn ? key : mn; mx = key > mx ? key : mx; seen = true;
      }
    }
    running += total;
  }
  if (seen) { atomicMin(&s_mn, mn); atomicMax(&s_mx, mx); atomicOr(&s_seen, 1u); }
  __syncthreads();
  if (tid == 0) {
    PageMetaDev m;
    m.uncomp_size = prefix + (rows - nnull) * j.pwidth;
    m.comp_size = m.uncomp_size;
    m.null_count = nnull;
    m.has_minmax = s_seen;
    m.mn = s_seen ? order_key_to_plain(s_mn, j.type) : 0;
    m.mx = s_seen ? order_key_to_plain(s_mx, j.type) : 0;
    m.head = prefix;
    m.enc = ENC_PLAIN;
    m.ndict = 0;
    m._pad = 0;
    meta[page] = m;
  }
}

// ------------------------------------------------------------------------------------------------ DELTA_BINARY_PACKED and dictionary pages
// Both stages read the PLAIN body page_body_kernel wrote (the statistics are the same for every encoding) and write the encoded body,
// level prefix included, into a second buffer.  They run on the pages of the columns that ask for them: CTA b encodes the page of row
// group b / ncl, column clist[b % ncl].
__device__ __forceinline__ uint64_t zigzag(int64_t v) { return (uint64_t(v) << 1) ^ uint64_t(v >> 63); }
__device__ __forceinline__ uint64_t load_any(const uint8_t* p, uint32_t w, bool aligned) {
  if (aligned) return w == 8 ? *reinterpret_cast<const uint64_t*>(p) : uint64_t(*reinterpret_cast<const uint32_t*>(p));
  uint64_t x = 0;
  for (uint32_t b = 0; b < w; b++) x |= uint64_t(p[b]) << (8 * b);
  return x;
}

// Bit-packs the 32 values v[0..31] (each < 2^bw) LSB first into 4 * bw bytes at q: lane k builds 32-bit word k (no atomics, any alignment).
__device__ __forceinline__ void pack32(const uint64_t* v, uint32_t bw, uint8_t* q, uint32_t lane) {
  for (uint32_t k = lane; k < bw; k += 32) {
    const uint32_t bit0 = 32 * k;
    uint32_t i = bit0 / bw, off = bit0 % bw, have = 0;
    uint64_t acc = 0;
    while (have < 32 && i < 32) { acc |= (v[i] >> off) << have; have += bw - off; off = 0; i++; }
    q[4 * k] = uint8_t(acc); q[4 * k + 1] = uint8_t(acc >> 8); q[4 * k + 2] = uint8_t(acc >> 16); q[4 * k + 3] = uint8_t(acc >> 24);
  }
}

// DELTA_BINARY_PACKED as parquet-rs and Arrow write it: <128><4><count><zigzag first>, then per block of 128 deltas <zigzag min delta>
// <4 bit widths> <miniblocks of 32>; miniblocks past the last delta are not stored (bit width 0), the last stored one is padded to 32.
// INT32 pages take 32-bit wrapping deltas (bit widths <= 32), INT64 pages 64-bit ones.  One pass = two blocks = one delta per thread:
// warp minima -> block minimum, warp maxima of delta - min -> miniblock bit width, thread 0 lays out the two blocks, warps pack.
__global__ void __launch_bounds__(kThreads) delta_encode_kernel(const PageJob* __restrict__ jobs, uint32_t ncols, const uint32_t* __restrict__ clist, uint32_t ncl,
                                                               const uint8_t* __restrict__ body, uint64_t bstride, uint8_t* __restrict__ enc, uint64_t estride,
                                                               PageMetaDev* __restrict__ meta) {
  __shared__ uint64_t s_v[kThreads];                   // delta - block minimum of this pass
  __shared__ long long s_min[kThreads / 32];
  __shared__ uint32_t s_bw[kThreads / 32], s_boff[2], s_run;
  const uint32_t page = (blockIdx.x / ncl) * ncols + clist[blockIdx.x % ncl];
  const PageJob j = jobs[page % ncols];
  if (j.dictionary && meta[page].enc == ENC_RLE_DICT) return;     // the chunk kept its dictionary
  const uint8_t* in = body + uint64_t(page) * bstride;
  uint8_t* out = enc + uint64_t(page) * estride;
  const uint32_t P = meta[page].head, w = j.pwidth, nv = (meta[page].uncomp_size - P) / w;
  const uint8_t* v = in + P;
  const bool al = (P & (w - 1)) == 0;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t i = tid; i < P; i += kThreads) out[i] = in[i];
  if (tid == 0) {
    uint8_t* q = out + P;
    const uint64_t x0 = nv ? load_any(v, w, al) : 0;
    uint32_t n = varint_put(q, uint64_t(128));
    n += varint_put(q + n, uint64_t(4));
    n += varint_put(q + n, uint64_t(nv));
    n += varint_put(q + n, zigzag(w == 8 ? int64_t(x0) : int64_t(int32_t(uint32_t(x0)))));
    s_run = P + n;
  }
  __syncthreads();
  const uint32_t nd = nv ? nv - 1 : 0;
  for (uint32_t base = 0; base < nd; base += kThreads) {
    const uint32_t d = base + tid;
    const bool has = d < nd;
    int64_t sd = 0;
    if (has) {
      const uint64_t a = load_any(v + size_t(d) * w, w, al), b = load_any(v + size_t(d + 1) * w, w, al);
      sd = w == 8 ? int64_t(b - a) : int64_t(int32_t(uint32_t(b) - uint32_t(a)));
    }
    long long m = has ? (long long)sd : LLONG_MAX;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const long long t = __shfl_xor_sync(0xffffffffu, m, o); m = t < m ? t : m; }
    if (lane == 0) s_min[warp] = m;
    __syncthreads();
    const uint32_t blk = uint32_t(tid) >> 7;
    long long mn = s_min[4 * blk];
    for (int x = 1; x < 4; x++) mn = s_min[4 * blk + x] < mn ? s_min[4 * blk + x] : mn;
    const uint64_t u = has ? uint64_t(sd) - uint64_t(mn) : 0;   // INT32: both in int32 range, so u < 2^32
    s_v[tid] = u;
    unsigned long long mx = u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, mx, o); mx = t > mx ? t : mx; }
    if (lane == 0) s_bw[warp] = mx ? uint32_t(64 - __clzll((long long)mx)) : 0u;
    __syncthreads();
    if (tid == 0) {
      uint32_t o = s_run;
      for (uint32_t b = 0; b < 2 && base + 128 * b < nd; b++) {
        long long bm = s_min[4 * b];
        for (int x = 1; x < 4; x++) bm = s_min[4 * b + x] < bm ? s_min[4 * b + x] : bm;
        s_boff[b] = o;
        o += varint_len(zigzag(bm)) + 4;
        for (uint32_t x = 0; x < 4; x++) if (base + 128 * b + 32 * x < nd) o += 4 * s_bw[4 * b + x];
      }
      s_run = o;
    }
    __syncthreads();
    const uint32_t b0 = base + 128 * blk;
    if (b0 < nd) {
      uint8_t* q = out + s_boff[blk];
      const uint64_t zz = zigzag(mn);
      const uint32_t zl = varint_len(zz);
      if ((tid & 127) == 0) {
        varint_put(q, zz);
        for (uint32_t x = 0; x < 4; x++) q[zl + x] = b0 + 32 * x < nd ? uint8_t(s_bw[4 * blk + x]) : uint8_t(0);
      }
      const uint32_t mi = uint32_t(warp) & 3u;
      if (b0 + 32 * mi < nd) {
        uint32_t off = zl + 4;
        for (uint32_t x = 0; x < mi; x++) off += 4 * s_bw[4 * blk + x];
        pack32(s_v + (tid & ~31), s_bw[warp], q + off, uint32_t(lane));
      }
    }
    __syncthreads();                                   // s_v, s_min and s_bw are rewritten by the next pass
  }
  if (tid == 0) {
    PageMetaDev& m = meta[page];
    m.uncomp_size = m.comp_size = s_run;
    m.head = P + (s_run - P) % 4;                      // the compressors see the stream as 4-byte words behind a literal head
    m.enc = ENC_DELTA_BINARY_PACKED;
  }
}

// Dictionary encoding as parquet-rs does it: keys are the physical bits (NaN payloads and +-0.0 are distinct entries), entries in order of
// first appearance.  A chunk whose dictionary page would exceed 1 MiB (parquet-rs's default dictionary_page_size_limit) keeps its
// `encoding` instead (PLAIN: the body is copied; DELTA: delta_encode_kernel runs on it next).
//   open addressing in per-page global scratch (2 x the values, rounded up to a power of two): atomicCAS claims a slot with the row,
//   a row finding its key lowers the slot's row with atomicMin, so every slot ends holding the FIRST row of its key whatever the thread
//   order; first rows are flagged, a prefix sum of the flags in row order gives the ids.
//   Data page: [levels][bit width][RLE / bit-packed hybrid]: aligned groups of 8 indices that hold one index become RLE runs (consecutive
//   groups of the same index merge), the rest bit-packed runs; run sizes by prefix sum, every group writes its own bytes.
constexpr uint32_t kDictLimit = 1u << 20;
constexpr uint32_t kEmpty = 0xffffffffu;

__host__ __device__ __forceinline__ uint32_t dict_table_size(uint32_t m) { uint32_t t = 2; while (t < 2 * m) t <<= 1; return t; }
__host__ __device__ __forceinline__ uint32_t dict_groups(uint32_t m) { return (m + 7) / 8 + 1; }
__host__ __device__ __forceinline__ uint64_t dict_scratch_bytes(uint32_t m) {
  return (uint64_t(dict_table_size(m)) + 2ull * m + 4ull * dict_groups(m) + 16) * 4;
}

__global__ void __launch_bounds__(kThreads) dict_encode_kernel(const PageJob* __restrict__ jobs, uint32_t ncols, const uint32_t* __restrict__ clist, uint32_t ncl,
                                                              const uint8_t* __restrict__ body, uint64_t bstride, uint8_t* __restrict__ enc, uint64_t estride,
                                                              uint8_t* __restrict__ dict, uint64_t dstride, PageMetaDev* __restrict__ meta, uint32_t dmeta0,
                                                              uint8_t* __restrict__ scratch, uint64_t sstride, uint32_t max_vals) {
  __shared__ uint32_t s_w[9];
  const uint32_t k = blockIdx.x, page = (k / ncl) * ncols + clist[k % ncl];
  const PageJob j = jobs[page % ncols];
  const uint8_t* in = body + uint64_t(page) * bstride;
  uint8_t* out = enc + uint64_t(page) * estride;
  uint8_t* dout = dict + uint64_t(k) * dstride;
  const uint32_t ulen = meta[page].uncomp_size, P = meta[page].head, w = j.pwidth, nv = (ulen - P) / w;
  const uint32_t T = dict_table_size(nv), lg = uint32_t(31 - __clz(int(T))), G = (nv + 7) / 8;
  const uint32_t M = max_vals, GM = dict_groups(M);
  uint32_t* owner = reinterpret_cast<uint32_t*>(scratch + uint64_t(k) * sstride);   // slot -> first row of its key, then its id
  uint32_t* slot = owner + dict_table_size(M);         // row -> slot
  uint32_t* idx = slot + M;                            // row -> first-row flag, then dictionary index
  uint32_t* gval = idx + M;                            // group -> its one index, or kEmpty
  uint32_t* run_of = gval + GM;
  uint32_t* run_pos = run_of + GM;
  uint32_t* run_out = run_pos + GM;
  const uint8_t* v = in + P;
  const bool al = (P & (w - 1)) == 0;
  const int tid = threadIdx.x;
  for (uint32_t i = tid; i < T; i += kThreads) owner[i] = kEmpty;
  __syncthreads();
  for (uint32_t i = tid; i < nv; i += kThreads) {
    const uint64_t x = load_any(v + size_t(i) * w, w, al);
    uint32_t h = uint32_t((x * 0x9E3779B97F4A7C15ull) >> (64 - lg));
    for (;;) {
      uint32_t o = owner[h];
      if (o == kEmpty) { o = atomicCAS(&owner[h], kEmpty, i); if (o == kEmpty) break; }
      if (load_any(v + size_t(o) * w, w, al) == x) { atomicMin(&owner[h], i); break; }
      h = (h + 1) & (T - 1);
    }
    slot[i] = h;
  }
  __syncthreads();
  for (uint32_t i = tid; i < nv; i += kThreads) idx[i] = owner[slot[i]] == i ? 1u : 0u;
  __syncthreads();
  uint32_t running = 0;
  for (uint32_t base = 0; base < nv; base += kThreads) {
    const uint32_t i = base + tid, f = i < nv ? idx[i] : 0u;
    uint32_t total;
    const uint32_t id = running + block_excl_scan<kThreads>(f, &total, s_w);
    if (f) {
      owner[slot[i]] = id;
      if (uint64_t(id + 1) * w <= kDictLimit) { const uint64_t x = load_any(v + size_t(i) * w, w, al); for (uint32_t b = 0; b < w; b++) dout[size_t(id) * w + b] = uint8_t(x >> (8 * b)); }
    }
    running += total;
  }
  const uint32_t ndict = running;
  __syncthreads();
  if (uint64_t(ndict) * w > kDictLimit) {              // dictionary refused: the chunk takes its fallback encoding
    if (j.encoding == ENC_PLAIN) for (uint32_t i = tid; i < ulen; i += kThreads) out[i] = in[i];
    if (tid == 0) { PageMetaDev& d = meta[dmeta0 + k]; d.uncomp_size = d.comp_size = 0; d.head = 0; }
    return;
  }
  for (uint32_t i = tid; i < nv; i += kThreads) idx[i] = owner[slot[i]];
  for (uint32_t i = tid; i < P; i += kThreads) out[i] = in[i];
  __syncthreads();
  const uint32_t bw = ndict > 1 ? uint32_t(32 - __clz(int(ndict - 1))) : 0u, vb = (bw + 7) / 8;
  for (uint32_t g = tid; g < G; g += kThreads) {
    const uint32_t a = 8 * g, b = a + 8 < nv ? a + 8 : nv, x = idx[a];
    bool uni = true;
    for (uint32_t i = a + 1; i < b; i++) uni = uni && idx[i] == x;
    gval[g] = uni ? x : kEmpty;
  }
  __syncthreads();
  // an RLE group: one index, and next to a group of the same index, or wide enough indices that a run of its own pays
  auto is_rle = [&](uint32_t g) { const uint32_t x = gval[g]; return x != kEmpty && (bw == 0 || bw >= 4 || (g > 0 && gval[g - 1] == x) || (g + 1 < G && gval[g + 1] == x)); };
  running = 0;
  for (uint32_t base = 0; base < G; base += kThreads) {
    const uint32_t g = base + tid;
    uint32_t st = 0;
    if (g < G) { const bool r = is_rle(g); st = (g == 0 || r != is_rle(g - 1) || (r && gval[g] != gval[g - 1])) ? 1u : 0u; }
    uint32_t total;
    const uint32_t r = running + block_excl_scan<kThreads>(st, &total, s_w) + st - 1;
    if (g < G) { run_of[g] = r; if (st) run_pos[r] = g; }
    running += total;
  }
  const uint32_t nruns = running;
  if (tid == 0) run_pos[nruns] = G;
  __syncthreads();
  auto run_vals = [&](uint32_t a, uint32_t b) { return (8 * b < nv ? 8 * b : nv) - 8 * a; };
  running = 0;
  for (uint32_t base = 0; base < nruns; base += kThreads) {
    const uint32_t r = base + tid;
    uint32_t sz = 0;
    if (r < nruns) {
      const uint32_t a = run_pos[r], b = run_pos[r + 1];
      sz = is_rle(a) ? varint_len(run_vals(a, b) << 1) + vb : varint_len(((b - a) << 1) | 1u) + (b - a) * bw;
    }
    uint32_t total;
    const uint32_t o = running + block_excl_scan<kThreads>(sz, &total, s_w);
    if (r < nruns) run_out[r] = o;
    running += total;
  }
  const uint32_t rl_bytes = running;
  __syncthreads();
  uint8_t* q0 = out + P + 1;
  if (tid == 0) out[P] = uint8_t(bw);
  for (uint32_t g = tid; g < G; g += kThreads) {
    const uint32_t r = run_of[g], a = run_pos[r], b = run_pos[r + 1];
    uint8_t* q = q0 + run_out[r];
    if (is_rle(a)) {
      if (g == a) { const uint32_t n = varint_put(q, run_vals(a, b) << 1); for (uint32_t x = 0; x < vb; x++) q[n + x] = uint8_t(gval[a] >> (8 * x)); }
    } else {
      const uint32_t hdr = ((b - a) << 1) | 1u;
      if (g == a) varint_put(q, hdr);
      q += varint_len(hdr) + (g - a) * bw;
      uint64_t acc = 0;
      uint32_t nb = 0, o = 0;
      for (uint32_t x = 0; x < 8; x++) {
        const uint32_t i = 8 * g + x;
        acc |= uint64_t(i < nv ? idx[i] : 0u) << nb;
        nb += bw;
        while (nb >= 8) { q[o++] = uint8_t(acc); acc >>= 8; nb -= 8; }
      }
    }
  }
  if (tid == 0) {
    PageMetaDev& m = meta[page];
    m.uncomp_size = m.comp_size = P + 1 + rl_bytes;
    m.head = P + (1 + rl_bytes) % 4;
    m.enc = ENC_RLE_DICT;
    m.ndict = ndict;
    PageMetaDev& d = meta[dmeta0 + k];
    d.uncomp_size = d.comp_size = ndict * w;
    d.head = 0;
  }
}

// ------------------------------------------------------------------------------------------------ bloom filters
// One block per (row group b / nb, column bcols[b % nb]): the split-block bloom filter of the chunk, hashed from the non-null values of
// the PLAIN body page_body_kernel wrote (whatever the chunk's final encoding).  Every value ORs its 8 mask words into its block; OR
// commutes, so the bitset does not depend on thread order.  smem: the bitset is built in shared memory (bbytes of it) and stored once;
// otherwise `bloom` is zeroed beforehand and the words are ORed in place.
__global__ void __launch_bounds__(kThreads) bloom_build_kernel(const PageJob* __restrict__ jobs, uint32_t ncols, const uint32_t* __restrict__ bcols,
                                                              uint32_t nb, const uint8_t* __restrict__ body, uint64_t bstride,
                                                              const PageMetaDev* __restrict__ meta, uint32_t R, uint32_t rg_rows,
                                                              uint8_t* __restrict__ bloom, uint32_t bbytes, int smem) {
  extern __shared__ uint32_t s_bits[];
  const uint32_t g = blockIdx.x / nb, c = bcols[blockIdx.x % nb];
  const uint64_t page = uint64_t(g) * ncols + c;
  const uint32_t nvals = rows_of_rg(g, R, rg_rows) - meta[page].null_count, w = jobs[c].pwidth;
  const uint8_t* v = body + page * bstride + meta[page].head;
  const bool al = (reinterpret_cast<uintptr_t>(v) & (w - 1)) == 0;
  const uint32_t nwords = bbytes / 4, nblocks = bbytes / 32;
  uint32_t* out = reinterpret_cast<uint32_t*>(bloom + uint64_t(blockIdx.x) * bbytes);
  uint32_t* bits = smem ? s_bits : out;
  if (smem) {
    for (uint32_t i = threadIdx.x; i < nwords; i += kThreads) s_bits[i] = 0;
    __syncthreads();
  }
  for (uint32_t i = threadIdx.x; i < nvals; i += kThreads) {
    const uint64_t x = load_any(v + size_t(i) * w, w, al);
    const uint64_t h = w == 8 ? bloom::xxh64_8(x) : bloom::xxh64_4(uint32_t(x));
    uint32_t* blk = bits + size_t(bloom::block_of(h, nblocks)) * 8;
#pragma unroll
    for (int k2 = 0; k2 < 8; k2++) atomicOr(blk + k2, bloom::mask_word(h, k2));
  }
  if (smem) {
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < nwords; i += kThreads) out[i] = s_bits[i];
  }
}

// ------------------------------------------------------------------------------------------------ Snappy compression
__device__ __forceinline__ uint32_t lit_header_len(uint32_t len) { return len <= 60 ? 1u : (len <= 0x100 ? 2u : (len <= 0x10000 ? 3u : (len <= 0x1000000 ? 4u : 5u))); }
__device__ __forceinline__ uint32_t lit_header_put(uint8_t* p, uint32_t len) {
  const uint32_t n = len - 1;
  if (len <= 60) { p[0] = uint8_t(n << 2); return 1; }
  const uint32_t nb = lit_header_len(len) - 1;
  p[0] = uint8_t((59 + nb) << 2);
  for (uint32_t i = 0; i < nb; i++) p[1 + i] = uint8_t(n >> (8 * i));
  return 1 + nb;
}
// copy of len (4..64) bytes at offset off (< 2048): 2-byte form when len <= 11, else the 3-byte form
__device__ __forceinline__ uint32_t copy_len(uint32_t len) { return len <= 11 ? 2u : 3u; }
__device__ __forceinline__ uint32_t copy_put(uint8_t* p, uint32_t len, uint32_t off) {
  if (len <= 11) { p[0] = uint8_t(1 | ((len - 4) << 2) | ((off >> 8) << 5)); p[1] = uint8_t(off); return 2; }
  p[0] = uint8_t(2 | ((len - 1) << 2)); p[1] = uint8_t(off); p[2] = uint8_t(off >> 8);
  return 3;
}

// class of value i relative to value i-1:  0 = no usable match (literal bytes), 1..4 = k low bytes differ, the 8-k high bytes
// are copied (8-byte values only), 9 = equal (run-length copy)
constexpr uint8_t kClsN = 0, kClsF = 9;

// One block per unit (page).  scratch: per unit `sstride` = snappy_scratch_bytes(max_vals) bytes: cls (u8), then run_of, run_pos and
// run_out (u32).
__host__ __device__ __forceinline__ uint64_t snappy_scratch_bytes(uint32_t m) { return ((uint64_t(m) + 15) & ~uint64_t(15)) + (uint64_t(m) * 3 + 4) * 4; }
__global__ void __launch_bounds__(kThreads) snappy_encode_kernel(const CompUnit* __restrict__ units, PageMetaDev* __restrict__ meta,
                                                                uint8_t* __restrict__ scratch, uint64_t sstride, uint32_t max_vals) {
  __shared__ uint32_t s_w[9];
  __shared__ uint32_t s_total;
  const CompUnit u = units[blockIdx.x];
  const uint32_t w = u.w;
  const uint8_t* in = u.in;
  uint8_t* out = u.out;
  const uint32_t ulen = meta[u.meta].uncomp_size;
  const uint32_t prefix = meta[u.meta].head;          // the level prefix (+ the odd bytes of a byte stream); 0 for a dictionary page
  const uint32_t nv = (ulen - prefix) / w;
  uint8_t* cls = scratch + uint64_t(blockIdx.x) * sstride;
  uint32_t* run_of = reinterpret_cast<uint32_t*>(cls + ((max_vals + 15u) & ~15u));   // run index of value i
  uint32_t* run_pos = run_of + max_vals;                                            // first value of run r, then: output offset of run r
  uint32_t* run_out = run_pos + max_vals + 1;
  const int tid = threadIdx.x;
  const uint8_t* v = in + prefix;
  const bool al = (prefix & (w - 1)) == 0;
  // ---- classes
  for (uint32_t i = tid; i < nv; i += kThreads) {
    uint8_t c = kClsN;
    if (i > 0) {
      const uint64_t x = load_any(v + size_t(i) * w, w, al) ^ load_any(v + size_t(i - 1) * w, w, al);
      if (x == 0) c = kClsF;
      else if (w == 8) { const uint32_t k = (71u - uint32_t(__clzll((long long)x))) / 8u; if (k <= 4) c = uint8_t(k); }   // k = differing low bytes
    }
    cls[i] = c;
  }
  __syncthreads();
  // ---- runs: a new run starts where the class changes; partial-match values are runs of their own
  uint32_t running = 0;
  for (uint32_t base = 0; base < nv; base += kThreads) {
    const uint32_t i = base + tid;
    uint32_t st = 0;
    if (i < nv) { const uint8_t c = cls[i]; st = (i == 0 || c != cls[i - 1] || (c >= 1 && c <= 4)) ? 1u : 0u; }
    uint32_t total;
    const uint32_t r = running + block_excl_scan<kThreads>(st, &total, s_w) + st - 1;      // inclusive - 1 = run index
    if (i < nv) { run_of[i] = r; if (st) run_pos[r] = i; }
    running += total;
  }
  const uint32_t nruns = running;
  if (tid == 0) run_pos[nruns] = nv;
  __syncthreads();
  // ---- emitted size of every run; the level prefix joins the first literal run
  const uint32_t pre = varint_len(ulen);                                   // varint(uncompressed length)
  running = 0;
  for (uint32_t base = 0; base < nruns + (nv == 0 ? 1u : 0u); base += kThreads) {
    const uint32_t r = base + tid;
    uint32_t sz = 0;
    if (nv == 0) { if (r == 0 && prefix) sz = lit_header_len(prefix) + prefix; }
    else if (r < nruns) {
      const uint32_t a = run_pos[r], b = run_pos[r + 1], c = cls[a];
      if (c == kClsN) { const uint32_t len = (b - a) * w + (r == 0 ? prefix : 0); sz = lit_header_len(len) + len; }
      else if (c == kClsF) { const uint32_t bytes = (b - a) * w, full = bytes / 64, rem = bytes % 64; sz = full * 3 + (rem ? copy_len(rem) : 0); }
      else sz = 1 + c + 2;                                                   // literal(c) + copy(8 - c, offset 8)
    }
    uint32_t total;
    const uint32_t o = running + block_excl_scan<kThreads>(sz, &total, s_w);
    if (r < nruns) run_out[r] = o;
    running += total;
  }
  if (tid == 0) s_total = running;
  __syncthreads();
  uint8_t* body_out = out + pre;
  if (tid == 0) {
    varint_put(out, ulen);
    meta[u.meta].comp_size = pre + s_total;
    if (nv == 0 && prefix) { const uint32_t h = lit_header_put(body_out, prefix); for (uint32_t i = 0; i < prefix; i++) body_out[h + i] = in[i]; }
  }
  if (nv == 0) return;
  // ---- emission: every value writes its own share
  {
    // the first run is a literal run (value 0 has no predecessor): header + level prefix
    const uint32_t len0 = (run_pos[1] - run_pos[0]) * w + prefix;
    const uint32_t h0 = lit_header_len(len0);
    if (tid == 0) lit_header_put(body_out, len0);
    for (uint32_t i = tid; i < prefix; i += kThreads) body_out[h0 + i] = in[i];
  }
  for (uint32_t i = tid; i < nv; i += kThreads) {
    const uint32_t r = run_of[i], a = run_pos[r], b = run_pos[r + 1];
    const uint8_t c = cls[i];
    uint8_t* o = body_out + run_out[r];
    if (c == kClsN) {
      const uint32_t len = (b - a) * w + (r == 0 ? prefix : 0);
      const uint32_t h = lit_header_len(len);
      if (i == a && r != 0) lit_header_put(o, len);
      uint8_t* q = o + h + (r == 0 ? prefix : 0) + (i - a) * w;
      for (uint32_t bb = 0; bb < w; bb++) q[bb] = v[size_t(i) * w + bb];
    } else if (c == kClsF) {
      const uint32_t per = 64 / w, qn = i - a;
      if (qn % per == 0) {
        const uint32_t left = (b - i) * w;
        copy_put(o + (qn / per) * 3, left < 64 ? left : 64, w);
      }
    } else {
      o[0] = uint8_t((uint32_t(c) - 1) << 2);
      for (uint32_t bb = 0; bb < c; bb++) o[1 + bb] = v[size_t(i) * w + bb];
      copy_put(o + 1 + c, 8 - c, 8);
    }
  }
}

// ------------------------------------------------------------------------------------------------ Zstandard compression
// One block per page, one frame per page: magic, Single_Segment descriptor with the smallest Frame_Content_Size field, no checksum.
// Blocks end on value ends: block 0 = level prefix + the values that fit in 128 KiB, every later block 128 KiB of values.
//
// Matches are found per value (width w): the previous value (offset w) when it is equal (the run becomes one match) or agrees in
// its w - k >= 3 high bytes (k literal bytes + a match of the high bytes), else the most recent earlier equal value of the page
// (hash of the value -> latest position, built chunk by chunk: chunk c looks up, then inserts with atomicMax, so a lookup only sees
// earlier chunks and the table does not depend on thread order; every candidate is confirmed by loading it).  A value continues the
// match of the value before it when both match at the same offset in the same block.  Everything else is a literal.
//
// Per block: raw literals; for each of the three sequence alphabets RLE mode when every code is the same, else the predefined table;
// an offset repeats the previous sequence's (repeat code 1) when its literal length is > 0 and it is not the block's first sequence.
// The FSE state walk is serial: one thread per (block, alphabet).  Codes, extra bits, bit positions (prefix sums), literal copies,
// headers and the bit emission (atomicOr into zeroed words: same bits whatever the thread order) are spread over the block.
constexpr uint32_t kZBlock = 128u << 10;
constexpr uint32_t kZMaxBlocks = 72;                  // pages of up to 1M values of 8 bytes (write_sst refuses larger row groups)
constexpr uint32_t kZMaxVals = 1000000;
constexpr int kZHashBits = 12;
constexpr uint8_t kZLit = 0xff;                       // value without a match

// per-page scratch of the encoder: mk (u8, the byte of the value where its match starts, kZLit = none), then u32 arrays
__host__ __device__ __forceinline__ uint64_t zstd_scratch_bytes(uint32_t m) {
  return ((uint64_t(m) + 15u) & ~uint64_t(15)) + uint64_t(m) * 4u * 7u + (uint64_t(m) + 1u) * 4u * 2u + uint64_t(m) * 2u * 3u + 64u;
}

struct ZFse {                                          // encoding side of one predefined FSE table
  uint8_t sym[64];                                     // symbol of every state (the decoder's spread)
  uint8_t cell[64];                                    // states of symbol x in increasing order: cell[cum[x] .. cum[x] + normp[x])
  uint8_t cum[53], normp[53], hb[53], cnt[53];         // normp = max(count, 1), hb = highbit(normp)
};

__device__ __forceinline__ int zhbit(uint32_t v) { return 31 - __clz(int(v)); }
__device__ __forceinline__ uint32_t zcode(const uint32_t* base, int n, uint32_t v) {      // largest code c with base[c] <= v
  int lo = 0, hi = n - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (base[mid] <= v) lo = mid; else hi = mid - 1; }
  return uint32_t(lo);
}

__global__ void __launch_bounds__(kThreads) zstd_encode_kernel(const CompUnit* __restrict__ units, PageMetaDev* __restrict__ meta,
                                                              uint8_t* __restrict__ scratch, uint64_t sstride, uint32_t max_vals) {
  __shared__ uint32_t s_w[9];
  __shared__ uint32_t s_hash[1 << kZHashBits];
  __shared__ ZFse s_fse[3];                            // literal length, match length, offset
  __shared__ uint32_t s_seq0[kZMaxBlocks + 1];         // first sequence of block b; [nblk] = number of sequences
  __shared__ uint32_t s_flags[kZMaxBlocks];            // bit t: codes of alphabet t differ within the block (predefined mode); bit 3: bytes differ
  __shared__ uint32_t s_init[kZMaxBlocks][3];          // final FSE states = the decoder's initial states
  __shared__ uint32_t s_kind[kZMaxBlocks], s_size[kZMaxBlocks], s_out[kZMaxBlocks], s_lit[kZMaxBlocks], s_bs[kZMaxBlocks], s_bsn[kZMaxBlocks];
  const CompUnit u = units[blockIdx.x];
  const uint32_t w = u.w;
  const uint8_t* in = u.in;
  uint8_t* out = u.out;
  const uint32_t ulen = meta[u.meta].uncomp_size;
  const uint32_t P = meta[u.meta].head;                // the level prefix (+ the odd bytes of a byte stream); 0 for a dictionary page
  const uint32_t nv = (ulen - P) / w;
  const uint32_t M = max_vals;
  uint8_t* mk = scratch + uint64_t(blockIdx.x) * sstride;
  uint32_t* dist = reinterpret_cast<uint32_t*>(mk + ((M + 15u) & ~15u));     // match offset in bytes of value i
  uint32_t* sx = dist + M;                             // sequences that start before value i
  uint32_t* mstart = sx + M;                           // sequence s: first matched byte, end of the match, offset
  uint32_t* mend = mstart + M;
  uint32_t* off = mend + M;
  uint32_t* code = off + M;                            // LL code | ML code << 8 | OF code << 16
  uint32_t* ov = code + M;                             // Offset_Value
  uint32_t* exbits = ov + M;                           // exclusive prefix sums over the sequences: bits, match bytes
  uint32_t* exml = exbits + M + 1;
  uint16_t* st = reinterpret_cast<uint16_t*>(exml + M + 1);   // [alphabet][s]: state bits of the step s -> s + 1 (count | value << 3)
  const int tid = threadIdx.x;
  const uint8_t* v = in + P;
  const bool aligned = (P & (w - 1)) == 0;
  const uint32_t V0 = (kZBlock - P) / w, Vb = kZBlock / w;    // values in block 0 / in every later block (write_sst keeps P < 128 KiB)
  const uint32_t nblk = nv > V0 ? 1 + (nv - V0 + Vb - 1) / Vb : 1;
  auto blk_of_val = [&](uint32_t i) -> uint32_t { return i < V0 ? 0u : 1u + (i - V0) / Vb; };
  auto first_val = [&](uint32_t b) -> uint32_t { return b == 0 ? 0u : V0 + (b - 1) * Vb; };
  auto blk_start = [&](uint32_t b) -> uint32_t { return b == 0 ? 0u : P + first_val(b) * w; };
  auto blk_end = [&](uint32_t b) -> uint32_t { return b + 1 == nblk ? ulen : P + (V0 + b * Vb) * w; };
  // ---- shared state; the three predefined tables as the decoder spreads them (RFC 8878 4.1.1)
  for (int i = tid; i < (1 << kZHashBits); i += kThreads) s_hash[i] = 0;
  // block 0 of a data page starts with the level-prefix length (< 2^24): never one repeated byte; a dictionary page's block 0 is simply
  // never an RLE block
  for (uint32_t b = tid; b < nblk; b += kThreads) s_flags[b] = b == 0 ? 8u : 0u;
  if (tid < 3) {
    ZFse& T = s_fse[tid];
    const int al = tid == 2 ? 5 : 6, ns = tid == 0 ? 36 : (tid == 1 ? 53 : 29), size = 1 << al;
    auto norm = [&](int s) { return tid == 0 ? zst::ll_default(s) : (tid == 1 ? zst::ml_default(s) : zst::of_default(s)); };
    int high = size;
    uint32_t cum = 0;
    for (int s = 0; s < ns; s++) {
      const int n = norm(s), np = n < 0 ? 1 : n;
      T.normp[s] = uint8_t(np); T.hb[s] = uint8_t(zhbit(uint32_t(np))); T.cum[s] = uint8_t(cum); T.cnt[s] = 0;
      cum += uint32_t(np);
      if (n == -1) T.sym[--high] = uint8_t(s);
    }
    const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
    int pos = 0;
    for (int s = 0; s < ns; s++) {
      for (int i = 0; i < norm(s); i++) {
        T.sym[pos] = uint8_t(s);
        do { pos = (pos + step) & mask; } while (pos >= high);
      }
    }
    for (int i = 0; i < size; i++) { const int s = T.sym[i]; T.cell[T.cum[s] + T.cnt[s]++] = uint8_t(i); }
  }
  __syncthreads();
  // ---- match of every value
  for (uint32_t base = 0; base < nv; base += kThreads) {
    const uint32_t i = base + tid;
    uint32_t h = 0;
    if (i < nv) {
      const uint64_t x = load_any(v + size_t(i) * w, w, aligned);
      h = uint32_t((x * 0x9E3779B97F4A7C15ull) >> (64 - kZHashBits));
      uint8_t m = kZLit;
      uint32_t d = 0, part = 0;
      if (i > 0) {
        const uint64_t dx = x ^ load_any(v + size_t(i - 1) * w, w, aligned);
        if (dx == 0) { m = 0; d = w; }
        else { const uint32_t k = uint32_t(63 - __clzll((long long)dx)) / 8u + 1u; if (k + 3 <= w) part = k; }     // k low bytes differ
      }
      if (m == kZLit) {
        const uint32_t j = s_hash[h];
        if (j && load_any(v + size_t(j - 1) * w, w, aligned) == x) { m = 0; d = (i - (j - 1)) * w; }
        else if (part) { m = uint8_t(part); d = w; }
      }
      mk[i] = m;
      dist[i] = d;
      const uint32_t b = blk_of_val(i);
      if (b > 0) {                                     // an RLE block: every value equals the block's first, whose bytes are all equal
        const uint64_t y = load_any(v + size_t(first_val(b)) * w, w, aligned);
        const uint64_t rep = (y & 0xffu) * 0x0101010101010101ull;
        if (x != y || y != (w == 8 ? rep : (rep & 0xffffffffull))) atomicOr(&s_flags[b], 8u);
      }
    }
    __syncthreads();
    if (i < nv) atomicMax(&s_hash[h], i + 1);
    __syncthreads();
  }
  // ---- sequences: one starts at every matched value that does not continue the match of the value before it
  auto cont = [&](uint32_t i) { return i > 0 && mk[i] == 0 && mk[i - 1] != kZLit && dist[i - 1] == dist[i] && blk_of_val(i) == blk_of_val(i - 1); };
  uint32_t running = 0;
  for (uint32_t base = 0; base < nv; base += kThreads) {
    const uint32_t i = base + tid;
    const uint32_t start = (i < nv && mk[i] != kZLit && !cont(i)) ? 1u : 0u;
    uint32_t total;
    const uint32_t ex = running + block_excl_scan<kThreads>(start, &total, s_w);
    if (i < nv) {
      sx[i] = ex;
      if (start) { mstart[ex] = P + i * w + mk[i]; off[ex] = dist[i]; }
      if (mk[i] != kZLit && (i + 1 == nv || !cont(i + 1))) mend[ex + start - 1] = P + (i + 1) * w;
      const uint32_t b = blk_of_val(i);
      if (b > 0 && i == first_val(b)) s_seq0[b] = ex;
    }
    running += total;
  }
  const uint32_t nseq = running;
  if (tid == 0) { s_seq0[0] = 0; s_seq0[nblk] = nseq; }
  __syncthreads();
  auto blk_of_seq = [&](uint32_t s) { return blk_of_val((mstart[s] - P) / w); };
  auto lit_len = [&](uint32_t s, uint32_t b) { return mstart[s] - (s == s_seq0[b] ? blk_start(b) : mend[s - 1]); };
  // ---- codes of every sequence, then the mode of each alphabet per block
  for (uint32_t s = tid; s < nseq; s += kThreads) {
    const uint32_t b = blk_of_seq(s), ll = lit_len(s, b), ml = mend[s] - mstart[s];
    const uint32_t o = (s != s_seq0[b] && ll > 0 && off[s - 1] == off[s]) ? 1u : off[s] + 3u;
    code[s] = zcode(zst::kLLBase, 36, ll) | (zcode(zst::kMLBase, 53, ml) << 8) | (uint32_t(zhbit(o)) << 16);
    ov[s] = o;
  }
  __syncthreads();
  for (uint32_t s = tid; s < nseq; s += kThreads) {
    const uint32_t b = blk_of_seq(s), d = code[s] ^ code[s_seq0[b]];
    const uint32_t f = ((d & 0xffu) ? 1u : 0u) | ((d & 0xff00u) ? 2u : 0u) | ((d & 0xff0000u) ? 4u : 0u);
    if (f) atomicOr(&s_flags[b], f);
  }
  __syncthreads();
  // ---- FSE state walk (serial): thread 3b + t encodes alphabet t of block b from its last sequence to its first
  if (uint32_t(tid) < 3 * nblk) {
    const uint32_t b = tid / 3, t = tid % 3, sb = s_seq0[b], se = s_seq0[b + 1];
    if (se > sb && ((s_flags[b] >> t) & 1u)) {
      const ZFse& T = s_fse[t];
      const uint32_t al = t == 2 ? 5 : 6, size = 1u << al, sh = 8 * t;
      uint16_t* stt = st + size_t(t) * M;
      uint32_t state = T.cell[T.cum[(code[se - 1] >> sh) & 0xffu]];
      stt[se - 1] = 0;
      for (uint32_t s = se - 1; s-- > sb;) {
        const uint32_t x = (code[s] >> sh) & 0xffu, X = state + size;
        uint32_t nb = al - T.hb[x];
        if ((X >> nb) < T.normp[x]) nb--;
        stt[s] = uint16_t(nb | ((X & ((1u << nb) - 1u)) << 3));
        state = T.cell[T.cum[x] + (X >> nb) - T.normp[x]];
      }
      s_init[b][t] = state;
    }
  }
  __syncthreads();
  // ---- bits of every sequence and match bytes: prefix sums
  running = 0;
  uint32_t running_ml = 0;
  for (uint32_t base = 0; base <= nseq; base += kThreads) {
    const uint32_t s = base + tid;
    uint32_t bits = 0, ml = 0;
    if (s < nseq) {
      const uint32_t c = code[s], fl = s_flags[blk_of_seq(s)];
      bits = zst::ll_bits(c & 0xffu) + zst::ml_bits((c >> 8) & 0xffu) + ((c >> 16) & 0xffu);
      for (uint32_t t = 0; t < 3; t++) if ((fl >> t) & 1u) bits += st[size_t(t) * M + s] & 7u;
      ml = mend[s] - mstart[s];
    }
    uint32_t total, total_ml;
    const uint32_t eb = running + block_excl_scan<kThreads>(bits, &total, s_w);
    const uint32_t em = running_ml + block_excl_scan<kThreads>(ml, &total_ml, s_w);
    if (s <= nseq) { exbits[s] = eb; exml[s] = em; }
    running += total;
    running_ml += total_ml;
  }
  __syncthreads();
  // ---- block type and size: RLE, compressed or raw, whichever is smallest
  for (uint32_t b = tid; b < nblk; b += kThreads) {
    const uint32_t sb = s_seq0[b], se = s_seq0[b + 1], n = se - sb, len = blk_end(b) - blk_start(b), fl = s_flags[b];
    uint32_t kind = 0, size = len;
    if (!(fl & 8u)) { kind = 1; size = 1; }
    else {
      const uint32_t lits = len - (exml[se] - exml[sb]);
      uint32_t c = (lits < 32 ? 1 : (lits < 4096 ? 2 : 3)) + lits;
      uint32_t nbytes = 0;
      if (n == 0) c += 1;
      else {
        const uint32_t bits = exbits[se] - exbits[sb] + ((fl & 1u) ? 6 : 0) + ((fl & 2u) ? 6 : 0) + ((fl & 4u) ? 5 : 0);
        nbytes = bits / 8 + 1;                         // + the end mark
        c += (n < 128 ? 1 : (n < 0x7f00 ? 2 : 3)) + 1 + (3 - __popc(fl & 7u)) + nbytes;
      }
      if (c < len) { kind = 2; size = c; s_bsn[b] = nbytes; }
    }
    s_kind[b] = kind;
    s_size[b] = size;
  }
  __syncthreads();
  const uint32_t fcs_flag = ulen < 256 ? 0u : (ulen < 65536u + 256u ? 1u : 2u);
  if (tid == 0) {
    uint32_t o = 4 + 1 + (fcs_flag == 0 ? 1 : (fcs_flag == 1 ? 2 : 4));
    for (uint32_t b = 0; b < nblk; b++) { s_out[b] = o; o += 3 + s_size[b]; }
    meta[u.meta].comp_size = o;
    const uint32_t fcs = fcs_flag == 1 ? ulen - 256 : ulen;
    const uint8_t hdr[5] = {0x28, 0xb5, 0x2f, 0xfd, uint8_t((fcs_flag << 6) | 0x20u)};     // Single_Segment, no checksum, no dictionary
    for (int i = 0; i < 5; i++) out[i] = hdr[i];
    for (uint32_t i = 0; i < (fcs_flag == 0 ? 1u : (fcs_flag == 1 ? 2u : 4u)); i++) out[5 + i] = uint8_t(fcs >> (8 * i));
  }
  __syncthreads();
  // ---- block, literals and sequences section headers
  for (uint32_t b = tid; b < nblk; b += kThreads) {
    const uint32_t kind = s_kind[b], bs = blk_start(b), len = blk_end(b) - bs;
    uint8_t* q = out + s_out[b];
    const uint32_t bh = (b + 1 == nblk ? 1u : 0u) | (kind << 1) | ((kind == 2 ? s_size[b] : len) << 3);
    q[0] = uint8_t(bh); q[1] = uint8_t(bh >> 8); q[2] = uint8_t(bh >> 16);
    q += 3;
    if (kind == 1) q[0] = in[bs];
    if (kind != 2) continue;
    const uint32_t sb = s_seq0[b], se = s_seq0[b + 1], n = se - sb, fl = s_flags[b];
    const uint32_t lits = len - (exml[se] - exml[sb]);
    if (lits < 32) *q++ = uint8_t(lits << 3);                                                  // Raw_Literals_Block
    else if (lits < 4096) { const uint32_t h = (1u << 2) | (lits << 4); *q++ = uint8_t(h); *q++ = uint8_t(h >> 8); }
    else { const uint32_t h = (3u << 2) | (lits << 4); *q++ = uint8_t(h); *q++ = uint8_t(h >> 8); *q++ = uint8_t(h >> 16); }
    s_lit[b] = uint32_t(q - out);
    q += lits;
    if (n < 128) *q++ = uint8_t(n);
    else if (n < 0x7f00) { *q++ = uint8_t((n >> 8) + 128); *q++ = uint8_t(n); }
    else { *q++ = 255; *q++ = uint8_t(n - 0x7f00); *q++ = uint8_t((n - 0x7f00) >> 8); }
    if (n) {
      const uint32_t c0 = code[sb];
      const uint32_t rle_ll = !(fl & 1u), rle_ml = !(fl & 2u), rle_of = !(fl & 4u);
      *q++ = uint8_t((rle_ll << 6) | (rle_of << 4) | (rle_ml << 2));                           // 0 = predefined, 1 = RLE
      if (rle_ll) *q++ = uint8_t(c0);
      if (rle_of) *q++ = uint8_t(c0 >> 16);
      if (rle_ml) *q++ = uint8_t(c0 >> 8);
    }
    s_bs[b] = uint32_t(q - out);
  }
  // ---- contents: raw blocks, literals of the compressed blocks; their bit streams are zeroed
  for (uint32_t b = 0; b < nblk; b++) {
    if (s_kind[b] == 0) {
      const uint32_t bs = blk_start(b), len = blk_end(b) - bs;
      for (uint32_t x = tid; x < len; x += kThreads) out[s_out[b] + 3 + x] = in[bs + x];
    }
  }
  __syncthreads();
  if (s_kind[0] == 2) for (uint32_t x = tid; x < P; x += kThreads) out[s_lit[0] + x] = in[x];
  for (uint32_t i = tid; i < nv; i += kThreads) {
    const uint32_t b = blk_of_val(i);
    const uint32_t m = mk[i], nl = m == kZLit ? w : m;
    if (s_kind[b] != 2 || nl == 0) continue;
    const uint32_t at = P + i * w - blk_start(b) - (exml[sx[i]] - exml[s_seq0[b]]);
    for (uint32_t k = 0; k < nl; k++) out[s_lit[b] + at + k] = v[size_t(i) * w + k];
  }
  for (uint32_t b = 0; b < nblk; b++) if (s_kind[b] == 2 && s_seq0[b + 1] > s_seq0[b]) for (uint32_t x = tid; x < s_bsn[b]; x += kThreads) out[s_bs[b] + x] = 0;
  __syncthreads();
  // ---- the bit streams.  Sequence s's bits start behind those of the later sequences of its block (the decoder reads backwards and
  //      meets sequence 0 first); low to high: state bits OF, ML, LL of the step to s + 1, then the extra bits LL, ML, OF
  uint32_t* wout = reinterpret_cast<uint32_t*>(out);
  auto put = [&](uint32_t b, uint32_t pos, uint32_t val, uint32_t n) {
    if (n == 0) return;
    const uint64_t g = uint64_t(s_bs[b]) * 8u + pos;
    const uint64_t x = uint64_t(val & ((1u << n) - 1u)) << (g & 31u);
    if (uint32_t(x)) atomicOr(&wout[g >> 5], uint32_t(x));
    if (x >> 32) atomicOr(&wout[(g >> 5) + 1], uint32_t(x >> 32));
  };
  for (uint32_t s = tid; s < nseq; s += kThreads) {
    const uint32_t b = blk_of_seq(s);
    if (s_kind[b] != 2) continue;
    const uint32_t fl = s_flags[b], c = code[s], llc = c & 0xffu, mlc = (c >> 8) & 0xffu, ofc = (c >> 16) & 0xffu;
    uint32_t pos = exbits[s_seq0[b + 1]] - exbits[s + 1];
    for (int t = 2; t >= 0; t--) {                     // OF, ML, LL
      if (!((fl >> t) & 1u)) continue;
      const uint32_t e = st[size_t(t) * M + s];
      put(b, pos, e >> 3, e & 7u);
      pos += e & 7u;
    }
    const uint32_t ll = lit_len(s, b), ml = mend[s] - mstart[s];
    put(b, pos, ll - zst::ll_base(llc), zst::ll_bits(llc)); pos += zst::ll_bits(llc);
    put(b, pos, ml - zst::ml_base(mlc), zst::ml_bits(mlc)); pos += zst::ml_bits(mlc);
    put(b, pos, ov[s] - (1u << ofc), ofc);
  }
  for (uint32_t b = tid; b < nblk; b += kThreads) {
    if (s_kind[b] != 2 || s_seq0[b + 1] == s_seq0[b]) continue;
    const uint32_t fl = s_flags[b];
    uint32_t pos = exbits[s_seq0[b + 1]] - exbits[s_seq0[b]];
    if (fl & 2u) { put(b, pos, s_init[b][1], 6); pos += 6; }     // initial states, ML, OF, LL (the decoder reads LL first)
    if (fl & 4u) { put(b, pos, s_init[b][2], 5); pos += 5; }
    if (fl & 1u) { put(b, pos, s_init[b][0], 6); pos += 6; }
    put(b, pos, 1, 1);                                 // end mark
  }
}

struct GatherDesc { const uint8_t* src; uint64_t dst_off; uint32_t bytes, _pad; };
__global__ void __launch_bounds__(kThreads) gather_pages_kernel(const GatherDesc* __restrict__ d, uint8_t* __restrict__ file) {
  const GatherDesc g = d[blockIdx.x];
  const uint8_t* s = g.src;
  uint8_t* t = file + g.dst_off;
  // destination-aligned 8-byte stores; the source word comes from two aligned loads + a funnel shift (any relative alignment)
  uint32_t head = uint32_t((8 - (reinterpret_cast<uintptr_t>(t) & 7)) & 7);
  if (head > g.bytes) head = g.bytes;
  if (threadIdx.x < head) t[threadIdx.x] = s[threadIdx.x];
  const uint32_t nwords = (g.bytes - head) >> 3;
  uint64_t* t8 = reinterpret_cast<uint64_t*>(t + head);
  const uint8_t* s0 = s + head;
  for (uint32_t wi = threadIdx.x; wi < nwords; wi += kThreads) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(s0 + (size_t(wi) << 3));
    const uint64_t* q = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
    const uint32_t sh = uint32_t(a & 7) * 8;
    const uint64_t lo = q[0];
    t8[wi] = sh ? ((lo >> sh) | (q[1] << (64 - sh))) : lo;
  }
  for (uint32_t i = head + (nwords << 3) + threadIdx.x; i < g.bytes; i += kThreads) t[i] = s[i];
}

// ------------------------------------------------------------------------------------------------ Thrift compact writer
class TOut {
 public:
  std::vector<uint8_t> b;
  std::vector<int> last;
  void uvar(uint64_t v) { while (v >= 0x80) { b.push_back(uint8_t(v | 0x80)); v >>= 7; } b.push_back(uint8_t(v)); }
  void svar(int64_t v) { uvar((uint64_t(v) << 1) ^ uint64_t(v >> 63)); }
  void begin() { last.push_back(0); }
  void end() { b.push_back(0); last.pop_back(); }
  void field(int id, int type) {
    const int delta = id - last.back();
    if (delta > 0 && delta <= 15) b.push_back(uint8_t((delta << 4) | type));
    else { b.push_back(uint8_t(type)); svar(id); }
    last.back() = id;
  }
  void i32(int id, int64_t v) { field(id, 5); svar(v); }
  void i64(int id, int64_t v) { field(id, 6); svar(v); }
  void boolean(int id, bool v) { field(id, v ? 1 : 2); }
  void binary(int id, const void* p, size_t n) { field(id, 8); uvar(n); const uint8_t* q = static_cast<const uint8_t*>(p); b.insert(b.end(), q, q + n); }
  void str(int id, const std::string& s) { binary(id, s.data(), s.size()); }
  void list(int id, int etype, size_t n) { field(id, 9); if (n < 15) b.push_back(uint8_t((n << 4) | etype)); else { b.push_back(uint8_t(0xf0 | etype)); uvar(n); } }
  void struct_field(int id) { field(id, 12); begin(); }
  void list_str(const std::string& s) { uvar(s.size()); b.insert(b.end(), s.begin(), s.end()); }
};

int converted_of(uint32_t t) {      // parquet ConvertedType for the integer types that need one (-1: none)
  switch (t) {
    case T_U8: return 11; case T_U16: return 12; case T_U32: return 13; case T_U64: return 14;
    case T_I8: return 15; case T_I16: return 16;
    default: return -1;
  }
}

// ColumnMetaData.encodings of a chunk from its data page's encoding: the levels' RLE, the values' encoding, and a dictionary's PLAIN page
void chunk_encodings(TOut& f, uint32_t enc) {
  if (enc == ENC_RLE_DICT) { f.list(2, 5, 3); f.svar(ENC_PLAIN); f.svar(ENC_RLE); f.svar(ENC_RLE_DICT); }
  else if (enc == ENC_DELTA_BINARY_PACKED) { f.list(2, 5, 2); f.svar(ENC_RLE); f.svar(ENC_DELTA_BINARY_PACKED); }
  else { f.list(2, 5, 2); f.svar(ENC_PLAIN); f.svar(ENC_RLE); }
}

constexpr uint32_t kBloomSmemMax = 128u << 10;      // larger bitsets are built with atomicOr on global words

// Per-page buffer strides and per-unit scratch sizes, for pages of up to max_vals values
struct PageStrides {
  uint64_t body, enc, dict, comp;      // PLAIN body, encoded body (DELTA / RLE_DICTIONARY), dictionary page, compressed page
  uint64_t snappy, zstd, dict_scratch;
  uint32_t cmax;                       // values (or 4-byte words) of the largest compressor input
};

// Where a page's bytes are: `in` uncompressed (a compressor reads it as a head + words of `w` bytes), `stored` as the file holds them
struct PageSrc { uint8_t* in; uint8_t* stored; uint32_t w; };

// A chunk's place in the file: [dictionary page header][dictionary page][data page header][data page]
struct ChunkPos {
  uint64_t off = 0, data_off = 0, uncomp = 0, comp = 0;   // uncomp / comp: page headers included
  int64_t dict_off = -1, bloom_off = -1;
  uint32_t bloom_len = 0;                                 // bloom filter header + bitset
};

template <typename T>
int upload(hg_engine* e, DevBuf* d, const std::vector<T>& v) {
  if (v.empty()) return HG_OK;
  CU_TRY(d->alloc(v.size() * sizeof(T), e->stream));
  return stage_upload(e, d->p, v.data(), v.size() * sizeof(T));
}

// One write_sst call.  Data page p = row group p / ncols, column p % ncols; dictionary page k = row group k / nd, column dcols[k % nd];
// bloom filter k = row group k / nb, column bcols[k % nb].
struct SstWrite {
  hg_engine* e;
  cudaStream_t s;
  const hg_schema_desc* schema;
  const ColIn* cols;
  uint32_t ncols, R;
  const WriteOpts& wo;
  const std::vector<hg_column_write_opts>& co;
  // plan
  uint32_t rg_rows = 0, nrg = 0, max_vals = 0, nd = 0, nb = 0;
  uint64_t npages = 0, ndu = 0;
  std::vector<PageJob> jobs;
  std::vector<uint32_t> dcols, ecols, bcols, dindex;   // columns with a dictionary, with DELTA (own or fallback), with a bloom filter
  bool any_zstd = false, any_codec = false;
  PageStrides st{};
  // alloc
  DevBuf d_jobs, d_body, d_enc, d_dict, d_comp, d_meta, d_scratch, d_clist, d_units, d_bloom, d_bcols;
  std::vector<CompUnit> su, zu;                       // Snappy / Zstd units: data page p -> comp slot p, dictionary page k -> npages + k
  // encode: data pages, then dictionary pages
  std::vector<PageMetaDev> meta;
  // lay_out
  std::vector<ChunkPos> chunk;
  std::vector<std::vector<uint8_t>> headers;
  std::vector<uint64_t> hdr_at;
  std::vector<GatherDesc> gd;
  uint64_t pos = 4;
  // footer
  TOut f;

  SstWrite(hg_engine* e, const hg_schema_desc* schema, const ColIn* cols, uint32_t R, const WriteOpts& wo)
      : e(e), s(e->stream), schema(schema), cols(cols), ncols(schema->num_columns), R(R), wo(wo), co(wo.cols) {}
  PageSrc data_src(uint64_t p) const {
    const uint32_t c = uint32_t(p % ncols);
    const bool encoded = co[c].encoding != ENC_PLAIN || co[c].dictionary;   // written to the second buffer, compressed as 4-byte words
    uint8_t* in = encoded ? d_enc.as<uint8_t>() + p * st.enc : d_body.as<uint8_t>() + p * st.body;
    return PageSrc{in, co[c].codec ? d_comp.as<uint8_t>() + p * st.comp : in, encoded ? 4u : jobs[c].pwidth};
  }

  PageSrc dict_src(uint64_t k) const {
    const uint32_t c = dcols[k % nd];
    uint8_t* in = d_dict.as<uint8_t>() + k * st.dict;
    return PageSrc{in, co[c].codec ? d_comp.as<uint8_t>() + (npages + k) * st.comp : in, jobs[c].pwidth};
  }

  // Page jobs, the column lists, buffer strides
  int plan() {
    rg_rows = wo.max_row_group_size;
    nrg = (R + rg_rows - 1) / rg_rows;
    npages = uint64_t(nrg) * ncols;
    jobs.resize(ncols);
    dindex.assign(ncols, 0);
    for (uint32_t c = 0; c < ncols; c++) {
      jobs[c] = PageJob{cols[c].vals, cols[c].valid, cols[c].type, cols[c].width, phys_width(phys_of(cols[c].type)), co[c].encoding, co[c].dictionary};
      if (co[c].dictionary) { dindex[c] = uint32_t(dcols.size()); dcols.push_back(c); }
      if (co[c].encoding == ENC_DELTA_BINARY_PACKED) ecols.push_back(c);
      if (co[c].bloom_filter) bcols.push_back(c);
      any_zstd = any_zstd || co[c].codec == CODEC_ZSTD;
      any_codec = any_codec || co[c].codec != CODEC_UNCOMPRESSED;
    }
    nd = uint32_t(dcols.size());
    nb = uint32_t(bcols.size());
    ndu = uint64_t(nrg) * nd;
    max_vals = std::min<uint32_t>(rg_rows, R ? R : 1);
    if (any_zstd && max_vals > kZMaxVals) return set_error(HG_ERR_UNSUPPORTED, "write: ZSTD pages hold at most 1,000,000 rows (max_row_group_size)");
    const bool any_encoded = nd || !ecols.empty();
    st.body = page_body_bytes(max_vals);
    // a DELTA body can exceed the PLAIN one: up to 14 header bytes per 128 values of 64-bit deltas, and the last miniblock padded to 32 values
    st.enc = any_encoded ? align64(st.body + st.body / 64 + 512) : 0;
    st.dict = nd ? align64(std::min<uint64_t>(uint64_t(max_vals) * 8, kDictLimit) + 16) : 0;
    const uint64_t src = std::max(st.body, std::max(st.enc, st.dict));
    // encoded bodies reach the compressors as 4-byte words: up to st.enc / 4 of them per page
    st.cmax = any_encoded ? std::max<uint32_t>(max_vals, uint32_t(st.enc / 4)) : max_vals;
    // Zstandard worst case: frame header (<= 9 bytes here) + 3 bytes per block on top of the page
    st.comp = any_zstd ? align64(src + 16 + 3 * (src / kZBlock + 2)) : src + 64;
    st.snappy = snappy_scratch_bytes(st.cmax);
    st.zstd = align64(zstd_scratch_bytes(st.cmax));
    st.dict_scratch = align64(dict_scratch_bytes(max_vals));
    return HG_OK;
  }

  // Device buffers, the compression units, and the uploads of the jobs, column lists, units and bloom filter columns
  int alloc() {
    meta.resize(npages + ndu);
    if (!npages) return HG_OK;
    CU_TRY(d_body.alloc(npages * st.body, s));
    CU_TRY(d_meta.alloc(meta.size() * sizeof(PageMetaDev), s));
    if (st.enc) CU_TRY(d_enc.alloc(npages * st.enc, s));
    if (nd) CU_TRY(d_dict.alloc(ndu * st.dict, s));
    if (any_codec) CU_TRY(d_comp.alloc((npages + ndu) * st.comp, s));
    if (nb) CU_TRY(d_bloom.alloc(uint64_t(nrg) * nb * wo.bloom_filter_bytes, s));
    auto add_unit = [&](uint32_t c, const PageSrc& src, uint64_t m) {
      if (co[c].codec) (co[c].codec == CODEC_SNAPPY ? su : zu).push_back(CompUnit{src.in, src.stored, uint32_t(m), src.w});
    };
    for (uint64_t p = 0; p < npages; p++) add_unit(uint32_t(p % ncols), data_src(p), p);
    for (uint64_t k = 0; k < ndu; k++) add_unit(dcols[k % nd], dict_src(k), npages + k);
    const uint64_t scratch = std::max(std::max(su.size() * st.snappy, zu.size() * st.zstd), ndu * st.dict_scratch);
    if (scratch) CU_TRY(d_scratch.alloc(scratch, s));
    std::vector<uint32_t> clist(dcols);
    clist.insert(clist.end(), ecols.begin(), ecols.end());
    std::vector<CompUnit> units(su);
    units.insert(units.end(), zu.begin(), zu.end());
    int rc = upload(e, &d_jobs, jobs);
    if (!rc) rc = upload(e, &d_clist, clist);
    if (!rc) rc = upload(e, &d_units, units);
    if (!rc) rc = upload(e, &d_bcols, bcols);
    return rc;
  }

  // The launches (page bodies, bloom filters, dictionary, DELTA, Snappy, Zstd), then the page metadata back to the host
  int encode() {
    if (!npages) return HG_OK;
    const PageJob* dj = d_jobs.as<PageJob>();
    uint8_t* body = d_body.as<uint8_t>();
    PageMetaDev* dm = d_meta.as<PageMetaDev>();
    page_body_kernel<<<uint32_t(npages), kThreads, 0, s>>>(dj, ncols, R, rg_rows, body, st.body, dm);
    e->launches++;
    if (nb) {
      const uint32_t bbytes = wo.bloom_filter_bytes;
      const uint64_t nbf = uint64_t(nrg) * nb;
      const int smem = bbytes <= kBloomSmemMax ? 1 : 0;
      if (!smem) CU_TRY(cudaMemsetAsync(d_bloom.p, 0, nbf * bbytes, s));
      else if (bbytes > (48u << 10)) CU_TRY(cudaFuncSetAttribute(bloom_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kBloomSmemMax)));
      bloom_build_kernel<<<uint32_t(nbf), kThreads, smem ? bbytes : 0, s>>>(dj, ncols, d_bcols.as<uint32_t>(), nb, body, st.body, dm, R, rg_rows,
                                                                             d_bloom.as<uint8_t>(), bbytes, smem);
      e->launches++;
    }
    if (ndu) {
      dict_encode_kernel<<<uint32_t(ndu), kThreads, 0, s>>>(dj, ncols, d_clist.as<uint32_t>(), nd, body, st.body, d_enc.as<uint8_t>(), st.enc,
                                                            d_dict.as<uint8_t>(), st.dict, dm, uint32_t(npages), d_scratch.as<uint8_t>(),
                                                            st.dict_scratch, max_vals);
      e->launches++;
    }
    if (!ecols.empty()) {
      delta_encode_kernel<<<uint32_t(uint64_t(nrg) * ecols.size()), kThreads, 0, s>>>(dj, ncols, d_clist.as<uint32_t>() + nd, uint32_t(ecols.size()),
                                                                                     body, st.body, d_enc.as<uint8_t>(), st.enc, dm);
      e->launches++;
    }
    if (!su.empty()) {
      snappy_encode_kernel<<<uint32_t(su.size()), kThreads, 0, s>>>(d_units.as<CompUnit>(), dm, d_scratch.as<uint8_t>(), st.snappy, st.cmax);
      e->launches++;
    }
    if (!zu.empty()) {
      zstd_encode_kernel<<<uint32_t(zu.size()), kThreads, 0, s>>>(d_units.as<CompUnit>() + su.size(), dm, d_scratch.as<uint8_t>(), st.zstd, st.cmax);
      e->launches++;
    }
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(meta.data(), d_meta.p, meta.size() * sizeof(PageMetaDev), cudaMemcpyDeviceToHost, s));
    CU_TRY(cudaStreamSynchronize(s));
    return HG_OK;
  }

  // A page header at pos, then `bytes` from src (gathered on the device)
  void put_page(std::vector<uint8_t>&& hdr, const uint8_t* src, uint32_t bytes) {
    hdr_at.push_back(pos);
    pos += hdr.size();
    headers.push_back(std::move(hdr));
    gd.push_back(GatherDesc{src, pos, bytes, 0});
    pos += bytes;
  }

  void add_page(ChunkPos* ch, TOut& hdr, const PageMetaDev& m, const uint8_t* src) {
    ch->uncomp += m.uncomp_size + hdr.b.size();
    ch->comp += m.comp_size + hdr.b.size();
    put_page(std::move(hdr.b), src, m.comp_size);
  }

  // Page headers and positions of every chunk, and the gather list
  void lay_out() {
    chunk.resize(npages);
    for (uint64_t p = 0; p < npages; p++) {
      const uint32_t g = uint32_t(p / ncols), c = uint32_t(p % ncols);
      ChunkPos& ch = chunk[p];
      ch.off = pos;
      if (meta[p].enc == ENC_RLE_DICT) {
        const uint64_t k = uint64_t(g) * nd + dindex[c];
        TOut t;
        t.begin();
        t.i32(1, PAGE_DICT);
        t.i32(2, meta[npages + k].uncomp_size);
        t.i32(3, meta[npages + k].comp_size);
        t.struct_field(7);                   // DictionaryPageHeader
        t.i32(1, meta[p].ndict);
        t.i32(2, ENC_PLAIN);
        t.end();
        t.end();
        ch.dict_off = int64_t(pos);
        add_page(&ch, t, meta[npages + k], dict_src(k).stored);
      }
      TOut t;
      t.begin();
      t.i32(1, PAGE_DATA);
      t.i32(2, meta[p].uncomp_size);
      t.i32(3, meta[p].comp_size);
      t.struct_field(5);                     // DataPageHeader
      t.i32(1, rows_of_rg(g, R, rg_rows));
      t.i32(2, meta[p].enc);
      t.i32(3, ENC_RLE);                     // definition levels
      t.i32(4, ENC_RLE);                     // repetition levels
      t.end();
      t.end();
      ch.data_off = pos;
      add_page(&ch, t, meta[p], data_src(p).stored);
      if (c + 1 == ncols) bloom_filters(g);
    }
  }

  // The row group's bloom filters follow its last chunk, in column order (parquet-rs's BloomFilterPosition::AfterRowGroup); they are not
  // part of any chunk's total_compressed_size
  void bloom_filters(uint32_t g) {
    const uint32_t bbytes = wo.bloom_filter_bytes;
    for (uint32_t i = 0; i < nb; i++) {
      TOut bh;
      bh.begin();
      bh.i32(1, bbytes);                     // numBytes
      bh.struct_field(2); bh.struct_field(1); bh.end(); bh.end();   // algorithm: BLOCK
      bh.struct_field(3); bh.struct_field(1); bh.end(); bh.end();   // hash: XXHASH
      bh.struct_field(4); bh.struct_field(1); bh.end(); bh.end();   // compression: UNCOMPRESSED
      bh.end();
      ChunkPos& ch = chunk[uint64_t(g) * ncols + bcols[i]];
      ch.bloom_off = int64_t(pos);
      ch.bloom_len = uint32_t(bh.b.size()) + bbytes;
      put_page(std::move(bh.b), d_bloom.as<uint8_t>() + (uint64_t(g) * nb + i) * bbytes, bbytes);
    }
  }

  // The FileMetaData
  void footer() {
    f.begin();
    f.i32(1, 1);                             // version (WriterVersion::PARQUET_1_0)
    f.list(2, 12, size_t(ncols) + 1);        // schema
    f.begin();
    f.str(4, "arrow_schema");
    f.i32(5, ncols);
    f.end();
    for (uint32_t c = 0; c < ncols; c++) {
      f.begin();
      f.i32(1, phys_of(cols[c].type));
      f.i32(3, 1);                           // OPTIONAL: every field of the reference's schemas is nullable
      f.str(4, col_name(schema, c));
      const int cv = converted_of(cols[c].type);
      if (cv >= 0) f.i32(6, cv);
      f.end();
    }
    f.i64(3, R);
    f.list(4, 12, nrg);
    for (uint32_t g = 0; g < nrg; g++) {
      f.begin();
      f.list(1, 12, ncols);
      uint64_t rg_uncomp = 0, rg_comp = 0;
      for (uint64_t p = uint64_t(g) * ncols; p < uint64_t(g + 1) * ncols; p++) {
        column_chunk(p);
        rg_uncomp += chunk[p].uncomp;
        rg_comp += chunk[p].comp;
      }
      f.i64(2, int64_t(rg_uncomp));
      f.i64(3, rows_of_rg(g, R, rg_rows));
      if (wo.sorting_columns) {
        f.list(4, 12, schema->num_primary_keys);
        for (uint32_t c = 0; c < schema->num_primary_keys; c++) { f.begin(); f.i32(1, c); f.boolean(2, false); f.boolean(3, true); f.end(); }
      }
      f.i64(5, int64_t(chunk[uint64_t(g) * ncols].off));
      f.i64(6, int64_t(rg_comp));
      f.field(7, 4); f.svar(g);              // ordinal (i16)
      f.end();
    }
    f.str(6, created_by());
    f.list(7, 12, ncols);                    // column_orders: TYPE_ORDER for every column (makes min_value / max_value usable)
    for (uint32_t c = 0; c < ncols; c++) { f.begin(); f.struct_field(1); f.end(); f.end(); }
    f.end();
  }

  void column_chunk(uint64_t p) {
    const uint32_t c = uint32_t(p % ncols);
    const ChunkPos& ch = chunk[p];
    const PageMetaDev& m = meta[p];
    f.begin();                               // ColumnChunk
    f.i64(2, int64_t(ch.off));               // file_offset
    f.struct_field(3);                       // ColumnMetaData
    f.i32(1, phys_of(cols[c].type));
    chunk_encodings(f, m.enc);
    f.list(3, 8, 1); f.list_str(col_name(schema, c));
    f.i32(4, int32_t(co[c].codec));
    f.i64(5, rows_of_rg(uint32_t(p / ncols), R, rg_rows));
    f.i64(6, int64_t(ch.uncomp));
    f.i64(7, int64_t(ch.comp));
    f.i64(9, int64_t(ch.data_off));          // data_page_offset
    if (ch.dict_off >= 0) f.i64(11, ch.dict_off);   // dictionary_page_offset
    f.struct_field(12);                      // Statistics
    f.i64(3, m.null_count);
    if (m.has_minmax) {
      f.binary(5, &m.mx, jobs[c].pwidth);    // max_value
      f.binary(6, &m.mn, jobs[c].pwidth);    // min_value
    }
    f.end();
    if (ch.bloom_off >= 0) {
      f.i64(14, ch.bloom_off);               // bloom_filter_offset
      f.i32(15, ch.bloom_len);               // bloom_filter_length: header + bitset
    }
    f.end();
    f.end();
  }

  // "(PLAIN, RLE levels, SNAPPY)" for the default configuration; otherwise every requested encoding and codec
  std::string created_by() const {
    bool plain = false, delta = false, dict = false, codec[7] = {false};
    for (uint32_t c = 0; c < ncols; c++) {
      dict = dict || co[c].dictionary;
      plain = plain || (!co[c].dictionary && co[c].encoding == ENC_PLAIN);
      delta = delta || (!co[c].dictionary && co[c].encoding == ENC_DELTA_BINARY_PACKED);
      codec[co[c].codec] = true;
    }
    std::string d = "horaedb_b200 GPU SST writer (";
    if (plain) d += "PLAIN, ";
    if (delta) d += "DELTA_BINARY_PACKED, ";
    if (dict) d += "RLE_DICTIONARY, ";
    d += "RLE levels";
    for (int k : {CODEC_UNCOMPRESSED, CODEC_SNAPPY, CODEC_ZSTD})
      if (codec[k]) d += std::string(", ") + (k == CODEC_SNAPPY ? "SNAPPY" : (k == CODEC_ZSTD ? "ZSTD" : "UNCOMPRESSED"));
    if (nb) d += ", bloom filters";
    return d + ")";
  }

  // The file image: pages gathered on the device and copied back once, then the page headers, the footer and the magic on the host
  int assemble(PinnedImage* out) {
    const uint64_t footer_off = pos;
    const uint64_t total = footer_off + f.b.size() + 8;
    if (total > 0xffffffffull) return set_error(HG_ERR_UNSUPPORTED, "output SST larger than 4 GiB (FileMeta.size is u32, sst.rs:155-160)");
    CU_TRY(cudaMallocHost(&out->p, total + 16));
    uint8_t* host = out->p;
    DevBuf d_file, d_gd;
    CU_TRY(d_file.alloc(total + 16, s));
    std::memcpy(host, "PAR1", 4);
    if (npages) {
      CU_TRY(d_gd.alloc(gd.size() * sizeof(GatherDesc), s));
      CU_TRY(cudaMemcpyAsync(d_gd.p, gd.data(), gd.size() * sizeof(GatherDesc), cudaMemcpyHostToDevice, s));
      gather_pages_kernel<<<uint32_t(gd.size()), kThreads, 0, s>>>(d_gd.as<GatherDesc>(), d_file.as<uint8_t>());
      e->launches++;
      CU_TRY(cudaMemcpyAsync(host + 4, d_file.as<uint8_t>() + 4, footer_off - 4, cudaMemcpyDeviceToHost, s));
      CU_TRY(cudaStreamSynchronize(s));
      for (size_t h = 0; h < headers.size(); h++) std::memcpy(host + hdr_at[h], headers[h].data(), headers[h].size());   // a few dozen bytes each
    }
    std::memcpy(host + footer_off, f.b.data(), f.b.size());
    const uint32_t flen = uint32_t(f.b.size());
    std::memcpy(host + footer_off + f.b.size(), &flen, 4);
    std::memcpy(host + footer_off + f.b.size() + 4, "PAR1", 4);
    out->size = total;
    e->stats.bytes_d2h += total;
    return HG_OK;
  }
};

}  // namespace

int resolve_write_opts(const hg_schema_desc* schema, const hg_write_props* props, WriteOpts* out) {
  const uint32_t n = schema->num_columns;
  auto known_codec = [](uint32_t k) { return k == CODEC_UNCOMPRESSED || k == CODEC_SNAPPY || k == CODEC_ZSTD; };
  if (!props->columns && !known_codec(props->compression))
    return set_error(HG_ERR_UNSUPPORTED, "write: only UNCOMPRESSED, SNAPPY and ZSTD pages are implemented");
  const uint32_t bb = props->bloom_filter_bytes;
  if (bb != 0 && (bb < bloom::kMinBytes || bb > bloom::kMaxBytes || (bb & (bb - 1)) != 0))
    return set_error(HG_ERR_INVALID, "write: bloom_filter_bytes " + std::to_string(bb) + " is not a power of two in [32, 128 MiB] (0 = 1 MiB)");
  out->cols.assign(n, hg_column_write_opts{ENC_PLAIN, 0, uint8_t(props->compression), 0});
  if (props->columns) out->cols.assign(props->columns, props->columns + n);
  out->max_row_group_size = props->max_row_group_size ? props->max_row_group_size : 8192;
  out->bloom_filter_bytes = bb ? bb : bloom::kDefaultBytes;
  out->sorting_columns = props->enable_sorting_columns != 0;
  for (uint32_t c = 0; c < n; c++) {
    const hg_column_write_opts& o = out->cols[c];
    const uint32_t t = schema->types[c];
    const std::string col = "write: column '" + col_name(schema, c) + "': ";
    if (t == T_BINARY) return set_error(HG_ERR_UNSUPPORTED, col + "Binary columns are not implemented in the GPU SST writer");
    if (!known_codec(o.codec))
      return set_error(HG_ERR_UNSUPPORTED, col + "codec " + std::to_string(o.codec) + " is not implemented (UNCOMPRESSED, SNAPPY and ZSTD are)");
    if (o.encoding != ENC_PLAIN && o.encoding != ENC_DELTA_BINARY_PACKED)
      return set_error(HG_ERR_UNSUPPORTED, col + "encoding " + std::to_string(o.encoding) + " is not implemented (PLAIN and DELTA_BINARY_PACKED are; "
                                               "a dictionary is the `dictionary` flag, with one of them as its fallback)");
    if (o.encoding == ENC_DELTA_BINARY_PACKED && type_is_float(t))
      return set_error(HG_ERR_UNSUPPORTED, col + "DELTA_BINARY_PACKED is defined for integer columns only");
    if (o.dictionary > 1) return set_error(HG_ERR_UNSUPPORTED, col + "dictionary must be 0 or 1");
    if (o.bloom_filter > 1) return set_error(HG_ERR_UNSUPPORTED, col + "bloom_filter must be 0 or 1");
  }
  return HG_OK;
}

int write_sst(hg_engine* e, const hg_schema_desc* schema, const ColIn* cols, uint32_t R, const WriteOpts& wo, PinnedImage* out) {
  SstWrite w(e, schema, cols, R, wo);
  int rc = w.plan();
  if (!rc) rc = w.alloc();
  if (!rc) rc = w.encode();
  if (rc) return rc;
  w.lay_out();
  w.footer();
  return w.assemble(out);
}

}  // namespace writer
}  // namespace horae
