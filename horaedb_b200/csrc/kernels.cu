// kernels.cu — general (materialising) pipeline of the columnar hot path, hand-written for sm_90a.
//
//   S2  snappy_chunks / zstd_chunks   : page decompress into the chunk's scratch (snappy.cu, zstd.cu; layout: chunk_scratch.h)
//       decode_chunks                 : RLE def levels, PLAIN / DELTA / dictionary values  (ParquetExec, read.rs:456-465)
//   S3  eval_predicates               : conjunction -> alive bytes                      (FilterExec, read.rs:467-469)
//       eval_binary_predicates        : its Binary predicates (byte compares), ANDed in
//   S4  build_records / merge_pass    : k-way merge on (pk.., __seq__)                  (SortPreservingMergeExec, read.rs:479-480)
//   S5  dedup_flags_*                 : PK-run boundaries                               (MergeStream::merge_batch, read.rs:289-343)
//   S6  keep last row of each run                                                       (LastValueOperator, operator.rs:39-44)
//   A1/A2 group_flags / reduce_groups : (group, ts/window) runs, sequential f64 sums    (types.rs:82-85 for the window)
//   A2  quantile_*                    : exact quantiles per group (hg_scan_quantile_aggregate)
//
// All of this is integer / byte work bounded by HBM bandwidth: kernels are grid-stride over the SMs, loads are
// coalesced and vectorised where the layout allows, no tensor cores.  Row counts that later kernels depend on stay on
// the device (d_m / d_r / d_g) so the pipeline never synchronises with the host between stages.
#include <cmath>

#include "kernels.h"
#include "block_scan.h"
#include "chunk_scratch.h"

namespace horae {
namespace k {

namespace {

constexpr int kThreads = 256;

// ---------------------------------------------------------------------------------------------- small device helpers
template <bool kCoherent>
__device__ __forceinline__ uint64_t ld64_any(const uint8_t* p) {
  uintptr_t a = reinterpret_cast<uintptr_t>(p);
  uint32_t sh = uint32_t(a & 7) * 8;
  const uint64_t* q = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
  uint64_t lo = kCoherent ? *reinterpret_cast<const volatile uint64_t*>(q) : __ldg(q);
  if (sh == 0) return lo;
  uint64_t hi = kCoherent ? *reinterpret_cast<const volatile uint64_t*>(q + 1) : __ldg(q + 1);
  return (lo >> sh) | (hi << (64 - sh));
}
__device__ __forceinline__ uint32_t ld32_any(const uint8_t* p) {
  uintptr_t a = reinterpret_cast<uintptr_t>(p);
  uint32_t sh = uint32_t(a & 3) * 8;
  const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  uint32_t lo = __ldg(q);
  if (sh == 0) return lo;
  uint32_t hi = __ldg(q + 1);
  return (lo >> sh) | (hi << (32 - sh));
}

__device__ __forceinline__ bool col_valid(const ColView& c, uint32_t row) { return c.valid == nullptr || c.valid[row] != 0; }

// ------------------------------------------------------------------------------------------------------- warp copy
// len bytes from src to dst, spread over the 32 lanes of the calling warp (kCoherent: src was written by this kernel)
template <bool kCoherent>
__device__ __forceinline__ void warp_copy(uint8_t* dst, const uint8_t* src, uint32_t len, int lane) {
  if (len < 32) {
    if (uint32_t(lane) < len) dst[lane] = kCoherent ? *reinterpret_cast<const volatile uint8_t*>(src + lane) : __ldg(src + lane);
    return;
  }
  uint32_t head = uint32_t((8 - (reinterpret_cast<uintptr_t>(dst) & 7)) & 7);
  if (uint32_t(lane) < head) dst[lane] = kCoherent ? *reinterpret_cast<const volatile uint8_t*>(src + lane) : __ldg(src + lane);
  uint32_t nwords = (len - head) >> 3;
  uint64_t* d8 = reinterpret_cast<uint64_t*>(dst + head);
  const uint8_t* s = src + head;
  for (uint32_t w = lane; w < nwords; w += 32) d8[w] = ld64_any<kCoherent>(s + (size_t(w) << 3));
  uint32_t done = head + (nwords << 3);
  uint32_t rem = len - done;
  if (uint32_t(lane) < rem)
    dst[done + lane] = kCoherent ? *reinterpret_cast<const volatile uint8_t*>(src + done + lane) : __ldg(src + done + lane);
}

// ------------------------------------------------------------------------------- def levels + PLAIN values -> columns
template <int OW>
__device__ __forceinline__ void store_val(void* out, uint32_t row, uint64_t v) {
  if (OW == 1) reinterpret_cast<uint8_t*>(out)[row] = uint8_t(v);
  else if (OW == 2) reinterpret_cast<uint16_t*>(out)[row] = uint16_t(v);
  else if (OW == 4) reinterpret_cast<uint32_t*>(out)[row] = uint32_t(v);
  else reinterpret_cast<uint64_t*>(out)[row] = v;
}
__device__ __forceinline__ void store_val_dyn(void* out, uint32_t ow, uint32_t row, uint64_t v) {
  switch (ow) {
    case 1: store_val<1>(out, row, v); break;
    case 2: store_val<2>(out, row, v); break;
    case 4: store_val<4>(out, row, v); break;
    default: store_val<8>(out, row, v);
  }
}

// ------------------------------------------------------------------------------------ DELTA_BINARY_PACKED -> PLAIN
// (Apache Parquet Encodings.md; a per-column option of the reference's writer, config.rs:54-75.)  One block per page:
// thread 0 walks the block headers (min delta, one bit width per miniblock), all threads unpack one block's deltas in
// parallel and a block-wide prefix sum turns them into values.  Sums wrap in the physical width, like the reference decoder.
__device__ __forceinline__ uint64_t block_incl_scan64(uint64_t v, uint64_t* total, uint64_t* s_w64 /*[9]*/) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint64_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t lo = __shfl_up_sync(0xffffffffu, uint32_t(inc), d), hi = __shfl_up_sync(0xffffffffu, uint32_t(inc >> 32), d);
    if (lane >= d) inc += (uint64_t(hi) << 32) | lo;
  }
  if (lane == 31) s_w64[w] = inc;
  __syncthreads();
  if (threadIdx.x == 0) { uint64_t run = 0; for (int x = 0; x < kThreads / 32; x++) { const uint64_t c = s_w64[x]; s_w64[x] = run; run += c; } s_w64[8] = run; }
  __syncthreads();
  const uint64_t r = s_w64[w] + inc;
  *total = s_w64[8];
  __syncthreads();
  return r;
}

// *end_pos (optional): bytes of [p, end) the encoded values occupy (what follows is the caller's: DELTA_LENGTH_BYTE_ARRAY data)
__device__ bool delta_decode_page(const uint8_t* p, const uint8_t* end, uint32_t pw, uint32_t max_out, uint8_t* out, uint32_t* count_out,
                                  uint32_t* end_pos = nullptr) {
  __shared__ uint64_t s_w64[9];
  __shared__ uint64_t s_min, s_cur;
  __shared__ uint32_t s_block, s_nmini, s_total, s_pos, s_ok;
  __shared__ uint32_t s_bw[64], s_moff[64];
  const int tid = threadIdx.x;
  auto varint = [&](uint32_t& pos, uint64_t* v) -> bool {
    uint64_t r = 0;
    for (int sh = 0; sh < 70; sh += 7) {
      if (p + pos >= end) return false;
      const uint8_t b = __ldg(p + pos++);
      r |= uint64_t(b & 0x7f) << sh;
      if (!(b & 0x80)) { *v = r; return true; }
    }
    return false;
  };
  if (tid == 0) {
    uint32_t pos = 0;
    uint64_t block = 0, nmini = 0, total = 0, zz = 0;
    bool ok = varint(pos, &block) && varint(pos, &nmini) && varint(pos, &total) && varint(pos, &zz);
    ok = ok && nmini > 0 && nmini <= 64 && block > 0 && block <= 65536 && block % nmini == 0 && (block / nmini) % 32 == 0 && total <= max_out;
    s_ok = ok;
    s_block = uint32_t(block); s_nmini = uint32_t(nmini); s_total = uint32_t(total); s_pos = pos;
    s_cur = (zz >> 1) ^ (0 - (zz & 1));
    if (ok && total > 0) {
      if (pw == 4) *reinterpret_cast<uint32_t*>(out) = uint32_t(s_cur); else *reinterpret_cast<uint64_t*>(out) = s_cur;
    }
  }
  __syncthreads();
  if (!s_ok) return false;
  const uint32_t total = s_total, block = s_block, nmini = s_nmini, per = block / nmini;
  __syncthreads();                                     // every thread has read the header before thread 0 reuses s_ok for the first block
  *count_out = total;
  uint32_t done = total ? 1u : 0u;
  while (done < total) {
    const uint32_t nvals = (total - done) < block ? (total - done) : block;
    if (tid == 0) {
      uint32_t pos = s_pos;
      uint64_t mz = 0;
      bool ok = varint(pos, &mz) && p + pos + nmini <= end;
      s_min = (mz >> 1) ^ (0 - (mz & 1));
      if (ok) {
        const uint32_t bwpos = pos;
        pos += nmini;
        for (uint32_t m = 0; m < nmini; m++) {
          const uint32_t b = __ldg(p + bwpos + m);
          s_bw[m] = b;
          s_moff[m] = pos;
          if (m * per < nvals) { if (b > 64) ok = false; pos += per * b / 8; }      // miniblocks past the last value are not stored
        }
        if (p + pos > end) ok = false;
      }
      s_pos = pos;
      s_ok = ok;
    }
    __syncthreads();
    if (!s_ok) return false;
    for (uint32_t base = 0; base < nvals; base += kThreads) {
      const uint32_t v = base + tid;
      uint64_t delta = 0;
      if (v < nvals) {
        const uint32_t m = v / per, j = v % per, b = s_bw[m];
        if (b) {
          const uint64_t bit = uint64_t(j) * b;
          const uint8_t* q = p + s_moff[m] + (bit >> 3);
          const uint32_t sh = uint32_t(bit & 7);
          const uint64_t lo = ld64_any<false>(q);
          uint64_t x = lo >> sh;
          if (sh && b + sh > 64) x |= uint64_t(__ldg(q + 8)) << (64 - sh);
          delta = b == 64 ? x : (x & ((1ull << b) - 1));
        }
        delta += s_min;
      }
      uint64_t tile_total;
      const uint64_t incl = block_incl_scan64(delta, &tile_total, s_w64);
      const uint64_t cur = s_cur;
      if (v < nvals) {
        const uint64_t val = cur + incl;
        if (pw == 4) reinterpret_cast<uint32_t*>(out)[done + v] = uint32_t(val); else reinterpret_cast<uint64_t*>(out)[done + v] = val;
      }
      __syncthreads();
      if (tid == 0) s_cur = cur + tile_total;
      __syncthreads();
    }
    done += nvals;
  }
  if (end_pos) *end_pos = s_pos;
  return true;
}

// ------------------------------------------------------------------------------------ RLE_DICTIONARY -> PLAIN
// Data page = [bit width][RLE / bit-packed hybrid runs of dictionary indices] (Parquet Encodings.md; enable_dict, config.rs:98-103).
// Thread 0 walks the run headers, all threads expand a run: out[i] = dict[index_i] as PLAIN values of width pw.  pw == 0: out[i] =
// index_i as a u32 (BYTE_ARRAY chunks, whose entries are resolved through the chunk's dictionary table).  max_out counts the page's
// NULL rows too, so the indices decoded can run into the padding of the last bit-packed group, which the spec leaves unspecified: the
// count returned stops at the first index outside the dictionary, and the caller fails the page only if a non-null row needs it.
__device__ bool dict_decode_page(const uint8_t* p, const uint8_t* end, uint32_t pw, uint32_t max_out, const uint8_t* dict, uint32_t dict_n,
                                 uint8_t* out, uint32_t* count_out) {
  __shared__ uint32_t s_kind, s_cnt, s_idx, s_pos, s_ok, s_first_bad;
  const int tid = threadIdx.x;
  if (tid == 0) { s_pos = 1; s_ok = p < end && __ldg(p) <= 32; s_first_bad = 0xffffffffu; }
  __syncthreads();
  if (!s_ok) return false;
  const uint32_t bw = __ldg(p);
  __syncthreads();                                     // every thread has read s_ok before thread 0 reuses it for the first run
  uint32_t done = 0;
  while (done < max_out) {
    if (tid == 0) {
      uint32_t pos = s_pos;
      bool ok = true;
      if (p + pos >= end) { s_cnt = 0; }
      else {
        uint64_t h = 0;
        int sh = 0;
        for (;;) {
          if (p + pos >= end || sh > 35) { ok = false; break; }
          const uint8_t b = __ldg(p + pos++);
          h |= uint64_t(b & 0x7f) << sh;
          sh += 7;
          if (!(b & 0x80)) break;
        }
        if (ok && (h & 1)) {                           // bit-packed run: (h >> 1) groups of 8 indices
          const uint64_t groups = h >> 1, bytes = groups * bw;
          if (groups == 0 || p + pos + bytes > end) ok = false;
          s_kind = 1; s_cnt = uint32_t(groups * 8 > 0xffffffffull ? 0xffffffffu : groups * 8); s_idx = pos;
          pos += uint32_t(bytes);
        } else if (ok) {                               // RLE run: count, then the index in ceil(bw / 8) bytes
          const uint32_t nb = (bw + 7) / 8;
          if ((h >> 1) == 0 || p + pos + nb > end) ok = false;
          uint32_t idx = 0;
          if (ok) for (uint32_t b = 0; b < nb; b++) idx |= uint32_t(__ldg(p + pos + b)) << (8 * b);
          s_kind = 0; s_cnt = uint32_t((h >> 1) > 0xffffffffull ? 0xffffffffu : (h >> 1)); s_idx = idx;
          pos += nb;
        }
      }
      s_pos = pos;
      s_ok = ok;
    }
    __syncthreads();
    if (!s_ok) return false;
    uint32_t cnt = s_cnt;
    if (cnt == 0) break;                               // index bytes exhausted
    if (cnt > max_out - done) cnt = max_out - done;
    const uint32_t kind = s_kind, ref = s_idx;
    for (uint32_t j = tid; j < cnt; j += kThreads) {
      uint32_t idx = ref;
      if (kind) {
        const uint64_t bit = uint64_t(j) * bw;
        const uint8_t* q = p + ref + (bit >> 3);
        const uint64_t x = ld64_any<false>(q) >> (bit & 7);
        idx = bw == 32 ? uint32_t(x) : uint32_t(x & ((1ull << bw) - 1));
      }
      if (idx >= dict_n) { atomicMin(&s_first_bad, done + j); idx = 0; }
      if (pw == 0) reinterpret_cast<uint32_t*>(out)[done + j] = idx;
      else if (dict_n) {
        if (pw == 4) reinterpret_cast<uint32_t*>(out)[done + j] = ld32_any(dict + size_t(idx) * 4);
        else reinterpret_cast<uint64_t*>(out)[done + j] = ld64_any<false>(dict + size_t(idx) * 8);
      }
    }
    done += cnt;
    __syncthreads();
  }
  __syncthreads();
  *count_out = done < s_first_bad ? done : s_first_bad;
  return true;
}

// ------------------------------------------------------------------------------------ BYTE_ARRAY dictionary / DELTA_BYTE_ARRAY
// A BYTE_ARRAY dictionary page is PLAIN byte arrays, [u32 length][bytes] each: one walk writes the (offset, length) of every entry to
// tab and returns their count, or ~0u when an entry runs past the page or the last one does not end exactly at the page end.  Thread 0
// only, out of line.
__device__ __noinline__ uint32_t index_byte_dict(const uint8_t* dict, uint32_t end, uint32_t* tab) {
  uint32_t pos = 0, n = 0;
  while (end - pos >= 4) {
    const uint32_t len = ld32_any(dict + pos);
    if (len > end - pos - 4) break;
    tab[2 * n] = pos + 4;
    tab[2 * n + 1] = len;
    n++;
    pos += 4 + len;
  }
  return pos == end ? n : ~0u;
}

// DELTA_BYTE_ARRAY (config.rs:54-75): [DELTA_BINARY_PACKED prefix lengths][DELTA_BINARY_PACKED suffix lengths][suffix bytes], all of
// the non-null values; value i = the first prefix[i] bytes of value i-1, then suffix i.  The values exist nowhere in the file, so the
// decode block only expands both runs into the page's scratch image (img: prefix [nv], suffix [nv]), checks them and sizes the page
// into *out; the host then places every page in one buffer and dba_materialise_kernel writes the values.  Rules: both runs cover
// exactly the non-null rows, prefix[0] == 0, prefix[i] <= length of value i-1, the suffix bytes fit in the page.  Every row is NULL
// until dba_materialise_kernel runs.  Returns false (and sizes the page 0, n 0) when a rule fails.  Called by the whole block.
__device__ __forceinline__ bool dba_size_page(const uint8_t* val_ptr, const uint8_t* page_end, uint32_t* img, uint32_t nv, uint32_t row,
                                           uint32_t ci, const ColSel& cs, bool all_valid, DbaPage* out) {
  __shared__ uint32_t s_warp[9], s_flag;
  __shared__ uint64_t s_w64[9];
  const int tid = threadIdx.x;
  uint32_t* pre = img;
  uint32_t* suf = img + nv;
  const uint8_t** optr = reinterpret_cast<const uint8_t**>(cs.out_vals);
  if (tid == 0) s_flag = 0;
  uint32_t c1 = 0, c2 = 0, u1 = 0, u2 = 0;
  bool ok = val_ptr <= page_end && delta_decode_page(val_ptr, page_end, 4, nv, reinterpret_cast<uint8_t*>(pre), &c1, &u1);
  __syncthreads();
  const uint8_t* sp = ok ? val_ptr + u1 : page_end;
  ok = ok && delta_decode_page(sp, page_end, 4, nv, reinterpret_cast<uint8_t*>(suf), &c2, &u2);
  __syncthreads();
  const uint8_t* data = ok ? sp + u2 : page_end;
  uint32_t nn = 0;
  for (uint32_t base = 0; base < nv; base += kThreads) {
    const uint32_t j = base + tid;
    const uint32_t v = (j < nv) ? (all_valid ? 1u : uint32_t(cs.out_valid[row + j] != 0)) : 0u;
    uint32_t tile_vals;
    (void)block_excl_scan<kThreads>(v, &tile_vals, s_warp);
    if (j < nv) { optr[row + j] = nullptr; cs.out_lens[row + j] = 0; }
    nn += tile_vals;
  }
  const bool go = ok && c1 == nn && c2 == nn;
  uint64_t total = 0, sufbytes = 0;
  for (uint32_t base = 0; go && base < nn; base += kThreads) {
    const uint32_t i = base + tid;
    uint64_t len = 0, s = 0;
    if (i < nn) {
      const uint32_t p = pre[i];
      s = suf[i];
      len = uint64_t(p) + s;
      if (i == 0 ? p != 0 : uint64_t(p) > uint64_t(pre[i - 1]) + suf[i - 1]) s_flag = 1;
    }
    uint64_t tile_len, tile_suf;
    (void)block_incl_scan64(len, &tile_len, s_w64);
    (void)block_incl_scan64(s, &tile_suf, s_w64);
    total += tile_len;
    sufbytes += tile_suf;
  }
  __syncthreads();
  const bool good = go && !s_flag && sufbytes <= uint64_t(page_end - data) && out != nullptr;
  __syncthreads();
  if (tid == 0 && out) {
    DbaPage d;
    d.lens = pre;
    d.suffix = data;
    d.bytes = good ? total : 0;
    d.out_off = 0;
    d.n = good ? nn : 0;
    d.nv = nv;
    d.row = row;
    d.ci = ci;
    *out = d;
  }
  return good;
}

// One block per selected chunk, 4 resident blocks per SM: that caps the kernel at 64 registers.  Without the bound ptxas picks 64 or
// 80 registers (3 blocks) depending on small changes anywhere in the kernel.
__global__ void __launch_bounds__(kThreads, 4) decode_chunks_kernel(const SstDev* __restrict__ ssts, const RgSel* __restrict__ sel,
                                                                    const ColSel* __restrict__ cols, int ncolsel,
                                                                    uint8_t* __restrict__ scratch, DbaPage* __restrict__ dba,
                                                                    const uint32_t* __restrict__ dba_base, int* err) {
  __shared__ uint32_t s_warp[9];
  __shared__ uint64_t s_w64b[9];
  __shared__ uint32_t s_kind, s_count, s_val, s_bad, s_dict_n;
  __shared__ const uint8_t* s_ptr;
  const int tid = threadIdx.x;
  uint32_t si = blockIdx.x / ncolsel;
  int ci = blockIdx.x % ncolsel;
  RgSel rs = sel[si];
  SstDev sst = ssts[rs.sst];
  const ChunkDev* chunks = sst.chunks + size_t(rs.rg) * sst.ncols;
  ColSel cs = cols[ci];
  ChunkDev ch = chunks[cs.col];
  const uint32_t pw = (ch.phys == 1 || ch.phys == 4) ? 4u : 8u;   // INT32/FLOAT : INT64/DOUBLE (BYTE_ARRAY: variable, handled apart)
  uint8_t* sc = scratch + (ch.scratch_bytes ? chunk_scratch_off(rs, chunks, cols, ci) : 0);
  // dictionary values (PLAIN): decompressed first in the scratch, or in place
  const uint8_t* dict = ch.dict_uncomp && ch.codec != CODEC_UNCOMPRESSED ? sc : sst.bytes + ch.dict_payload_off;
  const uint32_t dict_n = ch.dict_uncomp / pw;                       // fixed-width chunks only
  uint32_t* dtab = nullptr;                                          // BYTE_ARRAY dictionary: (offset, length) of every entry
  if (ch.phys == PT_BYTE_ARRAY && ch.dict_uncomp) dtab = reinterpret_cast<uint32_t*>(sc + dict_body_scratch(ch.codec, ch.dict_uncomp));
  sc += dict_scratch(ch.codec, ch.phys, ch.dict_uncomp);
  uint32_t row = rs.out_row;
  uint32_t ndba = 0;                                                 // DELTA_BYTE_ARRAY pages of this chunk so far
  if (tid == 0) {
    s_bad = 0;
    s_dict_n = 0;
    if (dtab) {
      const uint32_t nent = index_byte_dict(dict, ch.dict_uncomp, dtab);
      if (nent == ~0u) s_bad = 8; else s_dict_n = nent;
    }
  }
  __syncthreads();
  for (uint32_t p = 0; p < ch.num_pages; p++) {
    PageDev pg = sst.pages[ch.first_page + p];
    const uint32_t nv = pg.num_values;
    const uint8_t* payload = sst.bytes + pg.payload_off;
    const PageStream ps = page_stream(pg);
    const bool in_scratch = ch.codec != CODEC_UNCOMPRESSED && ps.compressed;   // the stream was decompressed to sc before this kernel
    const uint8_t* lv_ptr = nullptr;
    uint32_t lv_len = 0;
    const uint8_t* val_ptr;
    if (pg.page_type == PAGE_DATA_V2) { // V2: levels uncompressed in front, values optionally compressed
      lv_ptr = payload + pg.v2_rep_len;
      lv_len = pg.v2_def_len;
      val_ptr = in_scratch ? sc : payload + ps.skip;
    } else {                            // V1: [u32 len][levels][values], compressed as a whole
      const uint8_t* body = in_scratch ? sc : payload;
      if (ch.optional) {
        lv_len = ld32_any(body);
        lv_ptr = body + 4;
        val_ptr = body + 4 + lv_len;
      } else val_ptr = body;
    }
    // values available in this page (malformed pages must not make the decoder read past the page: ABI = HG_ERR_FORMAT)
    const uint8_t* page_end = in_scratch ? sc + ps.out : payload + pg.comp_size;
    uint32_t max_vals = val_ptr <= page_end ? uint32_t(size_t(page_end - val_ptr) / pw) : 0u;
    uint8_t* const img = sc + page_body_scratch(ch.codec, pg);         // the page's PLAIN image, or its length / index run
    if (pg.encoding == ENC_DELTA_BINARY_PACKED) {
      // DELTA_BINARY_PACKED: expand the values into the page's PLAIN image in scratch, then decode that like any PLAIN page
      uint32_t cnt = 0;
      const bool ok = val_ptr <= page_end && delta_decode_page(val_ptr, page_end, pw, nv, img, &cnt);
      __syncthreads();
      if (!ok) { if (tid == 0) s_bad = 4; cnt = 0; }
      val_ptr = img;
      max_vals = cnt;
      __syncthreads();
    } else if (ch.phys != PT_BYTE_ARRAY && (pg.encoding == ENC_RLE_DICT || pg.encoding == ENC_PLAIN_DICT)) {
      uint32_t cnt = 0;
      const bool ok = val_ptr <= page_end && dict_decode_page(val_ptr, page_end, pw, nv, dict, dict_n, img, &cnt);
      __syncthreads();
      if (!ok) { if (tid == 0) s_bad = 5; cnt = 0; }
      val_ptr = img;
      max_vals = cnt;
      __syncthreads();
    }

    bool all_valid = true;
    if (ch.optional) {
      // RLE / bit-packed hybrid, bit width 1.  Fast path: a single RLE run of 1s covering the page.
      const uint8_t* lp = lv_ptr;
      const uint8_t* lend = lv_ptr + lv_len;
      uint32_t i = 0;
      bool first = true;
      while (i < nv) {
        if (tid == 0) {
          uint32_t h = 0;
          int sh = 0;
          bool ok = false;
          while (lp < lend && sh < 35) {
            uint32_t b = __ldg(lp++);
            h |= (b & 0x7f) << sh;
            sh += 7;
            if (!(b & 0x80)) { ok = true; break; }
          }
          uint32_t kind = h & 1, cnt = h >> 1;
          if (kind) { cnt *= 8; s_ptr = lp; lp += (h >> 1); }
          else { s_val = (lp < lend) ? (__ldg(lp) & 1u) : 0u; lp += 1; }
          if (!ok || cnt == 0 || lp > lend) { s_bad = 1; cnt = nv; kind = 0; s_val = 1; }
          s_kind = kind;
          s_count = cnt;
        }
        __syncthreads();
        uint32_t kind = s_kind, cnt = s_count, val = s_val;
        const uint8_t* bp = s_ptr;
        if (cnt > nv - i) cnt = nv - i;
        if (first && kind == 0 && val == 1 && cnt == nv) { i = nv; __syncthreads(); break; }
        first = false;
        if (cs.out_valid == nullptr) {
          // no validity buffer (the chunk statistics say null_count = 0): the page stays all-valid whatever its run split — bit-packed
          // runs, many RLE runs — and only a level 0 is an error
          if (kind) { for (uint32_t j = tid; j < cnt; j += kThreads) if (!((__ldg(bp + (j >> 3)) >> (j & 7)) & 1u)) s_bad = 2; }
          else if (tid == 0 && val == 0) s_bad = 2;
        } else {
          all_valid = false;
          for (uint32_t j = tid; j < cnt; j += kThreads)
            cs.out_valid[row + i + j] = kind ? uint8_t((__ldg(bp + (j >> 3)) >> (j & 7)) & 1u) : uint8_t(val);
        }
        i += cnt;
        __syncthreads();
      }
    }
    if (ch.phys == 6 && pg.encoding == 6) {
      // BYTE_ARRAY, DELTA_LENGTH_BYTE_ARRAY (config.rs:54-75): [DELTA_BINARY_PACKED lengths of the non-null values][their bytes, back to
      // back].  The lengths expand into the page's scratch image, an exclusive scan turns them into offsets, and every row points at
      // its bytes in place.
      const uint8_t** optr = reinterpret_cast<const uint8_t**>(cs.out_vals);
      uint32_t* lens = reinterpret_cast<uint32_t*>(img);
      uint32_t cnt = 0, used = 0;
      bool ok = val_ptr <= page_end && delta_decode_page(val_ptr, page_end, 4, nv, reinterpret_cast<uint8_t*>(lens), &cnt, &used);
      __syncthreads();
      const uint8_t* data = val_ptr + used;
      const uint64_t room = ok && data <= page_end ? uint64_t(page_end - data) : 0;
      if (!ok || data > page_end) { if (tid == 0) s_bad = 7; cnt = 0; }
      if (all_valid && cs.out_valid) for (uint32_t j = tid; j < nv; j += kThreads) cs.out_valid[row + j] = 1;
      uint32_t run_vals = 0;                                  // non-null values before the current tile
      uint64_t run_off = 0;                                   // ... and their bytes
      for (uint32_t base = 0; base < nv; base += kThreads) {
        const uint32_t j = base + tid;
        const uint32_t v = (j < nv) ? (all_valid ? 1u : uint32_t(cs.out_valid[row + j] != 0)) : 0u;
        uint32_t tile_vals;
        const uint32_t kidx = run_vals + block_excl_scan<kThreads>(v, &tile_vals, s_warp);
        const uint64_t len = (v && kidx < cnt) ? lens[kidx] : 0;
        uint64_t tile_bytes;
        const uint64_t incl = block_incl_scan64(len, &tile_bytes, s_w64b);
        if (j < nv) {
          const uint64_t off = run_off + incl - len;
          if (v && (kidx >= cnt || off + len > room)) { s_bad = 7; optr[row + j] = nullptr; cs.out_lens[row + j] = 0; }
          else if (v) { optr[row + j] = data + off; cs.out_lens[row + j] = uint32_t(len); }
          else { optr[row + j] = nullptr; cs.out_lens[row + j] = 0; }
        }
        run_vals += tile_vals;
        run_off += tile_bytes;
        __syncthreads();
      }
    } else if (ch.phys == 6 && (pg.encoding == 8 || pg.encoding == 2)) {
      // BYTE_ARRAY, dictionary indices (enable_dict, storage.rs:271-283): the indices expand into the page's scratch image, and every
      // non-null row points at its entry in the dictionary page (in place, or in the decompression scratch).
      const uint8_t** optr = reinterpret_cast<const uint8_t**>(cs.out_vals);
      uint32_t* idxs = reinterpret_cast<uint32_t*>(img);
      uint32_t cnt = 0;
      const bool ok = val_ptr <= page_end && dict_decode_page(val_ptr, page_end, 0, nv, nullptr, s_dict_n, reinterpret_cast<uint8_t*>(idxs), &cnt);
      __syncthreads();
      if (!ok) { if (tid == 0) s_bad = 8; cnt = 0; }
      if (all_valid && cs.out_valid) for (uint32_t j = tid; j < nv; j += kThreads) cs.out_valid[row + j] = 1;
      uint32_t run_vals = 0;
      for (uint32_t base = 0; base < nv; base += kThreads) {
        const uint32_t j = base + tid;
        const uint32_t v = (j < nv) ? (all_valid ? 1u : uint32_t(cs.out_valid[row + j] != 0)) : 0u;
        uint32_t tile_vals;
        const uint32_t kidx = run_vals + block_excl_scan<kThreads>(v, &tile_vals, s_warp);
        if (j < nv) {
          if (v && kidx < cnt) {
            const uint32_t e = idxs[kidx];                    // < s_dict_n: dict_decode_page counts checked indices only
            optr[row + j] = dict + dtab[2 * e];
            cs.out_lens[row + j] = dtab[2 * e + 1];
          } else {
            if (v) s_bad = 8;
            optr[row + j] = nullptr;
            cs.out_lens[row + j] = 0;
          }
        }
        run_vals += tile_vals;
      }
    } else if (ch.phys == 6 && pg.encoding == 7) {
      // BYTE_ARRAY, DELTA_BYTE_ARRAY: sized here, written by dba_materialise_kernel (see dba_size_page)
      if (all_valid && cs.out_valid) for (uint32_t j = tid; j < nv; j += kThreads) cs.out_valid[row + j] = 1;
      const bool good = dba_size_page(val_ptr, page_end, reinterpret_cast<uint32_t*>(img), nv, row, uint32_t(ci), cs, all_valid,
                                      dba ? dba + dba_base[blockIdx.x] + ndba : nullptr);
      if (tid == 0 && !good) s_bad = 9;
      ndba++;
    } else if (ch.phys == 6) {
      // BYTE_ARRAY, PLAIN: [u32 length][bytes] per non-null value — a serial walk (a value's position depends on every length
      // before it); Binary values of this engine's tables are few and large (batched payloads), one thread does it.  Rows point
      // at their bytes in place (page payload or decompression scratch): nothing is copied here.
      const uint8_t** optr = reinterpret_cast<const uint8_t**>(cs.out_vals);
      if (tid == 0) {
        const uint8_t* p = val_ptr;
        bool bad = p > page_end;
        for (uint32_t j = 0; j < nv && !bad; j++) {
          const bool v = all_valid || cs.out_valid[row + j] != 0;
          if (v) {
            if (p + 4 > page_end) { bad = true; break; }
            const uint32_t len = ld32_any(p);
            if (len > uint32_t(page_end - p - 4)) { bad = true; break; }
            optr[row + j] = p + 4;
            cs.out_lens[row + j] = len;
            p += 4 + size_t(len);
          } else { optr[row + j] = nullptr; cs.out_lens[row + j] = 0; }
        }
        if (bad) s_bad = 6;
      }
      if (all_valid && cs.out_valid) for (uint32_t j = tid; j < nv; j += kThreads) cs.out_valid[row + j] = 1;
    } else if (all_valid && nv > max_vals) {
      if (tid == 0) s_bad = 3;
    } else if (all_valid) {
      if (pw == 8) {
        for (uint32_t j = tid; j < nv; j += kThreads) store_val<8>(cs.out_vals, row + j, ld64_any<false>(val_ptr + size_t(j) * 8));
      } else {
        for (uint32_t j = tid; j < nv; j += kThreads) store_val_dyn(cs.out_vals, cs.out_width, row + j, ld32_any(val_ptr + size_t(j) * 4));
      }
      if (cs.out_valid) for (uint32_t j = tid; j < nv; j += kThreads) cs.out_valid[row + j] = 1;
    } else if (cs.out_valid) {
      uint32_t running = 0;
      for (uint32_t base = 0; base < nv; base += kThreads) {
        uint32_t j = base + tid;
        uint32_t v = (j < nv) ? cs.out_valid[row + j] : 0;
        uint32_t total;
        uint32_t kidx = running + block_excl_scan<kThreads>(v, &total, s_warp);
        if (j < nv) {
          uint64_t x = 0;
          if (v && kidx >= max_vals) { s_bad = 3; v = 0; }
          if (v) x = pw == 8 ? ld64_any<false>(val_ptr + size_t(kidx) * 8) : uint64_t(ld32_any(val_ptr + size_t(kidx) * 4));
          store_val_dyn(cs.out_vals, cs.out_width, row + j, x);
        }
        running += total;
      }
    }
    row += nv;
    sc = img + page_image_scratch(pg);                                 // the next page's part
    __syncthreads();
  }
  if (tid == 0 && s_bad) atomicExch(err, 110 + int(s_bad));
}

// ----------------------------------------------------------------------------------- DELTA_BYTE_ARRAY -> values
// One warp per page, values in order, like the serial-per-stream decompressors: value i's prefix is copied from value i-1, which is
// already in the output, then its suffix from the page; each copy is spread over the lanes and a __syncwarp orders value i's bytes
// before value i+1 reads them.  Pages are independent, so they spread over the machine.  Rows point into `out`.
constexpr int kDbaWarps = 8;
__global__ void __launch_bounds__(kDbaWarps * 32) dba_materialise_kernel(const DbaPage* __restrict__ pages, uint32_t npages,
                                                                         const ColSel* __restrict__ cols, uint8_t* out) {
  const int lane = threadIdx.x & 31;
  const uint32_t w = blockIdx.x * kDbaWarps + (threadIdx.x >> 5);
  if (w >= npages) return;
  const DbaPage d = pages[w];
  const ColSel cs = cols[d.ci];
  const uint8_t** optr = reinterpret_cast<const uint8_t**>(cs.out_vals);
  const uint32_t* pre = d.lens;
  const uint32_t* suf = d.lens + d.nv;
  uint8_t* const dst = out + d.out_off;
  const uint32_t below = (1u << lane) - 1u;
  uint32_t k = 0, o = 0, so = 0, prev = 0;     // values done, their bytes, suffix bytes consumed, offset of the last value
  for (uint32_t base = 0; base < d.nv; base += 32) {
    const uint32_t j = base + uint32_t(lane);
    const bool v = j < d.nv && cs.out_valid[d.row + j] != 0;
    const uint32_t m = __ballot_sync(0xffffffffu, v);
    const uint32_t kk = k + uint32_t(__popc(m & below));
    const bool has = v && kk < d.n;                        // n == 0: the page failed validation, its rows stay NULL
    const uint32_t p = has ? pre[kk] : 0u, s = has ? suf[kk] : 0u, len = p + s;
    const uint32_t lincl = warp_incl_scan(len, lane), sincl = warp_incl_scan(s, lane);
    const uint32_t myo = o + lincl - len, myso = so + sincl - s;
    if (has) { optr[d.row + j] = dst + myo; cs.out_lens[d.row + j] = len; }
    for (uint32_t mm = __ballot_sync(0xffffffffu, has); mm; mm &= mm - 1) {
      const int src = __ffs(int(mm)) - 1;
      const uint32_t vp = __shfl_sync(0xffffffffu, p, src), vs = __shfl_sync(0xffffffffu, s, src);
      const uint32_t vo = __shfl_sync(0xffffffffu, myo, src), vso = __shfl_sync(0xffffffffu, myso, src);
      if (vp) warp_copy<true>(dst + vo, dst + prev, vp, lane);
      if (vs) warp_copy<false>(dst + vo + vp, d.suffix + vso, vs, lane);
      prev = vo;
      __syncwarp();
    }
    k += uint32_t(__popc(m));
    o += __shfl_sync(0xffffffffu, lincl, 31);
    so += __shfl_sync(0xffffffffu, sincl, 31);
  }
}

// ---------------------------------------------------------------------------------------------------- S3: predicates
__global__ void __launch_bounds__(kThreads) eval_predicates_kernel(PredSet preds, uint32_t n, uint8_t* __restrict__ alive) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    bool keep = true;
    for (int p = 0; p < preds.n && keep; p++) {
      const PredDev& pd = preds.p[p];
      if (!col_valid(pd.col, i)) { keep = false; break; }      // NULL => false
      const uint64_t v = widen(col_raw(pd.col, i), pd.col.type);
      const uint32_t cls = cmp_class(pd.col.type);
      if (pd.op == OP_IN) {
        bool any = false;
        for (uint32_t j = 0; j < pd.n_in && !any; j++) any = cmp_widened(v, pd.in_list[j], cls) == 0;
        keep = any;
        continue;
      }
      keep = op_holds(cmp_widened(v, pd.lit, cls), pd.op);
    }
    alive[i] = keep ? 1 : 0;
  }
}

// Binary predicates on the decoded rows (a pointer and a length each): one u64 compare of the rows' and the literals' 8-byte keys decides
// most rows; the bytes behind the key are read only when the keys tie.  The literal table is read through shared memory.  and_alive: the
// rows eval_predicates_kernel (launched before) failed stay failed.
__global__ void __launch_bounds__(kThreads) eval_binary_predicates_kernel(BinPredSet preds, uint32_t n, int and_alive, uint8_t* __restrict__ alive) {
  extern __shared__ BinLitDev s_lits[];
  for (uint32_t j = threadIdx.x; j < preds.n_lits; j += kThreads) s_lits[j] = preds.lits[j];
  __syncthreads();
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    bool keep = !and_alive || alive[i] != 0;
    for (int p = 0; p < preds.n && keep; p++) {
      const BinPredDev& pd = preds.p[p];
      if (!col_valid(pd.col, i)) { keep = false; break; }      // NULL => false
      const uint8_t* v = reinterpret_cast<const uint8_t* const*>(pd.col.vals)[i];
      const uint32_t len = pd.col.lens[i];
      const uint64_t key = bytes_key(v, len);
      if (pd.op == OP_IN) {
        bool any = false;
        for (uint32_t j = pd.first; j < pd.first + pd.n_lit && !any; j++) {
          const BinLitDev& l = s_lits[j];
          any = l.key == key && l.len == len && (len <= 8 || cmp_bytes_keyed(key, v, len, l.key, l.p, l.len) == 0);
        }
        keep = any;
        continue;
      }
      const BinLitDev& l = s_lits[pd.first];
      keep = op_holds(cmp_bytes_keyed(key, v, len, l.key, l.p, l.len), pd.op);
    }
    alive[i] = keep ? 1 : 0;
  }
}

// The tiled search over a sorted, unique set of order keys that eval_in_set_kernel and group_map_kernel share.  A block takes a tile of
// kInSetTile rows and reduces their keys to a minimum and a maximum (stage_set_slice); two binary searches over the set give the slice
// those rows can match: a few keys on a sorted key column, where a tile spans few series.  The block stages the slice in shared memory —
// all of it when it has at most kInSetSmemKeys keys, else every step-th key as splitters — and every row does one binary search there
// (find_in_slice), finished inside one step-long run of the set in global memory (L2) when its splitter is not the key itself.
struct SetSlice { uint32_t lo, hi, step, ns; };   // keys[lo, hi) staged as s_keys[i] = keys[lo + i * step], i < ns; hi == lo: empty

// Block-wide; every thread passes the minimum and maximum of its own live keys (mn > mx when it has none).  An empty slice stages nothing.
__device__ __forceinline__ SetSlice stage_set_slice(const uint64_t* __restrict__ keys, uint32_t n, uint64_t mn, uint64_t mx, uint64_t* s_keys,
                                                    uint64_t* s_mn, uint64_t* s_mx, uint32_t* s_slice) {
  constexpr int kWarps = kThreads / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const uint64_t a = __shfl_xor_sync(0xffffffffu, mn, d), b = __shfl_xor_sync(0xffffffffu, mx, d);
    mn = a < mn ? a : mn;
    mx = b > mx ? b : mx;
  }
  if (lane == 0) { s_mn[warp] = mn; s_mx[warp] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kWarps; w++) { mn = s_mn[w] < mn ? s_mn[w] : mn; mx = s_mx[w] > mx ? s_mx[w] : mx; }
    uint32_t lo = 0, hi = 0;
    if (mn <= mx) key_set_slice(keys, n, mn, mx, &lo, &hi);          // mn > mx: no row of the tile is live
    s_slice[0] = lo;
    s_slice[1] = hi;
  }
  __syncthreads();
  SetSlice sl{s_slice[0], s_slice[1], 0, 0};
  const uint32_t len = sl.hi - sl.lo;
  if (len == 0) return sl;
  sl.step = (len + kInSetSmemKeys - 1) / kInSetSmemKeys;
  sl.ns = (len + sl.step - 1) / sl.step;
  for (uint32_t i = threadIdx.x; i < sl.ns; i += kThreads) s_keys[i] = keys[sl.lo + i * sl.step];
  __syncthreads();
  return sl;
}

// The position of `key` in keys[] when the staged slice holds it, else kNotInSet
constexpr uint32_t kNotInSet = 0xffffffffu;
__device__ __forceinline__ uint32_t find_in_slice(const uint64_t* __restrict__ keys, const SetSlice& sl, const uint64_t* s_keys, uint64_t key) {
  uint32_t a = 0, b = sl.ns;                                           // the last staged key <= key
  while (a < b) { const uint32_t m = (a + b) >> 1; if (s_keys[m] <= key) a = m + 1; else b = m; }
  if (a == 0) return kNotInSet;
  const uint32_t at = sl.lo + (a - 1) * sl.step;
  if (s_keys[a - 1] == key) return at;
  if (sl.step > 1) {                                                   // splitters: the run between this one and the next
    const uint32_t end = min(sl.lo + a * sl.step, sl.hi);
    uint32_t g = at + 1, ge = end;
    while (g < ge) { const uint32_t m = (g + ge) >> 1; if (__ldg(keys + m) < key) g = m + 1; else ge = m; }
    if (g < end && __ldg(keys + g) == key) return g;
  }
  return kNotInSet;
}

// OP_IN_SET predicates on the decoded rows, one tile of kInSetTile rows per block step; per predicate the tile's rows still alive
// search the slice of the set they can match.  An empty slice fails the tile at once.  and_alive: rows the kernels launched before
// failed stay failed.
__global__ void __launch_bounds__(kThreads) eval_in_set_kernel(InSetPreds preds, uint32_t n, int and_alive, uint8_t* __restrict__ alive) {
  constexpr int kPer = int(kInSetTile) / kThreads;
  constexpr int kWarps = kThreads / 32;
  __shared__ uint64_t s_keys[kInSetSmemKeys];
  __shared__ uint64_t s_mn[kWarps], s_mx[kWarps];
  __shared__ uint32_t s_slice[2];
  const uint32_t ntiles = (n + kInSetTile - 1) / kInSetTile;
  for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const uint32_t base = tile * kInSetTile + threadIdx.x;           // row j of this thread: base + j * kThreads
    bool keep[kPer];
#pragma unroll
    for (int j = 0; j < kPer; j++) {
      const uint32_t row = base + uint32_t(j) * kThreads;
      keep[j] = row < n && (!and_alive || alive[row] != 0);
    }
    for (int p = 0; p < preds.n; p++) {
      const InSetDev& pd = preds.p[p];
      uint64_t key[kPer];
      uint64_t mn = ~0ull, mx = 0;
#pragma unroll
      for (int j = 0; j < kPer; j++) {
        const uint32_t row = base + uint32_t(j) * kThreads;
        key[j] = 0;
        if (!keep[j]) continue;
        if (!col_valid(pd.col, row)) { keep[j] = false; continue; }        // NULL => false
        key[j] = order_key(widen(col_raw(pd.col, row), pd.col.type), pd.col.type);
        mn = key[j] < mn ? key[j] : mn;
        mx = key[j] > mx ? key[j] : mx;
      }
      const SetSlice sl = stage_set_slice(pd.keys, pd.n, mn, mx, s_keys, s_mn, s_mx, s_slice);
      if (sl.hi == sl.lo) {
#pragma unroll
        for (int j = 0; j < kPer; j++) keep[j] = false;
        break;
      }
#pragma unroll
      for (int j = 0; j < kPer; j++)
        if (keep[j]) keep[j] = find_in_slice(pd.keys, sl, s_keys, key[j]) != kNotInSet;
    }
#pragma unroll
    for (int j = 0; j < kPer; j++) {
      const uint32_t row = base + uint32_t(j) * kThreads;
      if (row < n) alive[row] = keep[j] ? 1 : 0;
    }
  }
}

// The group of every deduplicated row of a by-map aggregate: out[rows[t]] = groups[i] where keys[i] is the order key of the row's key
// column, t < *d_r.  Every such row passed `key IN_SET keys` (the same keys), so a NULL or a key the set lacks is an internal error:
// the row's group stays unwritten and *err becomes kErrGroupMapMiss.
__global__ void __launch_bounds__(kThreads) group_map_kernel(ColView col, const uint32_t* __restrict__ rows, const uint32_t* d_r,
                                                            const uint64_t* __restrict__ keys, const uint32_t* __restrict__ groups, uint32_t n_keys,
                                                            uint32_t* __restrict__ out, int* err) {
  constexpr int kPer = int(kInSetTile) / kThreads;
  constexpr int kWarps = kThreads / 32;
  __shared__ uint64_t s_keys[kInSetSmemKeys];
  __shared__ uint64_t s_mn[kWarps], s_mx[kWarps];
  __shared__ uint32_t s_slice[2];
  const uint32_t r = *d_r, ntiles = (r + kInSetTile - 1) / kInSetTile;
  for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const uint32_t base = tile * kInSetTile + threadIdx.x;
    uint32_t row[kPer];
    uint64_t key[kPer];
    bool live[kPer];
    uint64_t mn = ~0ull, mx = 0;
    bool miss = false;
#pragma unroll
    for (int j = 0; j < kPer; j++) {
      const uint32_t t = base + uint32_t(j) * kThreads;
      live[j] = t < r;
      row[j] = live[j] ? rows[t] : 0;
      key[j] = 0;
      if (!live[j]) continue;
      if (!col_valid(col, row[j])) { live[j] = false; miss = true; continue; }
      key[j] = order_key(widen(col_raw(col, row[j]), col.type), col.type);
      mn = key[j] < mn ? key[j] : mn;
      mx = key[j] > mx ? key[j] : mx;
    }
    const SetSlice sl = stage_set_slice(keys, n_keys, mn, mx, s_keys, s_mn, s_mx, s_slice);
#pragma unroll
    for (int j = 0; j < kPer; j++) {
      if (!live[j]) continue;
      const uint32_t at = sl.hi == sl.lo ? kNotInSet : find_in_slice(keys, sl, s_keys, key[j]);
      if (at == kNotInSet) miss = true;
      else out[row[j]] = groups[at];
    }
    if (miss) atomicExch(err, kErrGroupMapMiss);
  }
}

// --------------------------------------------------------------------------------------------- stream compaction
constexpr int kCompactPerThread = 8;
constexpr int kCompactTile = kThreads * kCompactPerThread;  // 2048 flags per block

__device__ __forceinline__ uint32_t load_flags8(const uint8_t* flags, uint32_t base, uint32_t n, uint8_t f[8]) {
  uint32_t cnt = 0;
  if (base + 8 <= n) {
    uint2 v = *reinterpret_cast<const uint2*>(flags + base);   // base is a multiple of 8 and flags is 256B-aligned
    uint32_t w0 = v.x, w1 = v.y;
#pragma unroll
    for (int i = 0; i < 4; i++) { f[i] = (w0 >> (8 * i)) & 0xff ? 1 : 0; f[4 + i] = (w1 >> (8 * i)) & 0xff ? 1 : 0; }
  } else {
#pragma unroll
    for (int i = 0; i < 8; i++) f[i] = (base + i < n && flags[base + i]) ? 1 : 0;
  }
#pragma unroll
  for (int i = 0; i < 8; i++) cnt += f[i];
  return cnt;
}

__global__ void __launch_bounds__(kThreads) compact_count_kernel(const uint8_t* __restrict__ flags, uint32_t n, uint32_t* __restrict__ sums) {
  __shared__ uint32_t s_warp[9];
  uint32_t nblocks = (n + kCompactTile - 1) / kCompactTile;
  for (uint32_t b = blockIdx.x; b < nblocks; b += gridDim.x) {
    uint8_t f[8];
    uint32_t base = b * kCompactTile + threadIdx.x * kCompactPerThread;
    uint32_t c = base < n ? load_flags8(flags, base, n, f) : 0;
    uint32_t total;
    (void)block_excl_scan<kThreads>(c, &total, s_warp);
    if (threadIdx.x == 0) sums[b] = total;
  }
}

// single block: exclusive scan of sums[0..nb) in place; total -> *d_total (optional)
__global__ void __launch_bounds__(1024) compact_scan_sums_kernel(uint32_t* sums, uint32_t nb, uint32_t* d_total) {
  __shared__ uint32_t s_w[1024 / 32 + 1];
  uint32_t carry = 0;
  for (uint32_t base = 0; base < nb; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    uint32_t total;
    const uint32_t ex = block_excl_scan<1024>(i < nb ? sums[i] : 0, &total, s_w);
    if (i < nb) sums[i] = carry + ex;
    carry += total;
  }
  if (d_total && threadIdx.x == 0) *d_total = carry;
}

__global__ void __launch_bounds__(kThreads) compact_write_kernel(const uint8_t* __restrict__ flags, uint32_t n,
                                                                const uint32_t* __restrict__ sums, uint32_t* __restrict__ out_idx) {
  __shared__ uint32_t s_warp[9];
  uint32_t nblocks = (n + kCompactTile - 1) / kCompactTile;
  for (uint32_t b = blockIdx.x; b < nblocks; b += gridDim.x) {
    uint8_t f[8];
    uint32_t base = b * kCompactTile + threadIdx.x * kCompactPerThread;
    uint32_t c = base < n ? load_flags8(flags, base, n, f) : 0;
    uint32_t total;
    uint32_t o = sums[b] + block_excl_scan<kThreads>(c, &total, s_warp);
    if (c) {
#pragma unroll
      for (int i = 0; i < 8; i++) if (f[i]) out_idx[o++] = base + i;
    }
  }
}

// ------------------------------------------------------------------------------------------------ S4: merge records
__global__ void survivor_run_starts_kernel(const uint32_t* __restrict__ surv, const uint32_t* d_m,
                                           const uint32_t* __restrict__ file_base, int k, uint32_t* run_start) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > k) return;
  uint32_t m = *d_m;
  if (f == k) { run_start[k] = m; return; }
  uint32_t target = file_base[f];
  uint32_t lo = 0, hi = m;             // first survivor index with row >= file_base[f]
  if (surv == nullptr) lo = target < m ? target : m;
  else while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (surv[mid] < target) lo = mid + 1; else hi = mid; }
  run_start[f] = lo;
}

__device__ __forceinline__ void pk_key128(const PkSet& pk, uint32_t row, uint64_t* hi, uint64_t* lo) {
  unsigned __int128 key = 0;
  for (int c = 0; c < pk.n; c++) {
    uint32_t w = pk.c[c].width;
    uint64_t v = col_raw(pk.c[c], row);
    if (type_is_signed(pk.c[c].type)) v ^= (uint64_t(1) << (8 * w - 1));   // order-preserving map to unsigned
    key = (key << (8 * w)) | v;
  }
  *hi = uint64_t(key >> 64);
  *lo = uint64_t(key);
}

__global__ void __launch_bounds__(kThreads) build_records_kernel(PkSet pk, ColView seq, const uint32_t* __restrict__ surv,
                                                                const uint32_t* d_m, SortRec* __restrict__ rec) {
  uint32_t m = *d_m;
  for (uint32_t j = blockIdx.x * kThreads + threadIdx.x; j < m; j += gridDim.x * kThreads) {
    uint32_t row = surv ? surv[j] : j;
    SortRec r;
    pk_key128(pk, row, &r.k0, &r.k1);
    // ASC NULLS FIRST: null sorts before every value.  (value + 1, NULL = 0) would wrap at u64 max onto NULL, so the validity goes
    // above the row id instead: it decides between equal seq values before the row does
    const bool v = col_valid(seq, row);
    r.seq = v ? col_raw(seq, row) : 0;
    r.row = (uint64_t(v) << 32) | row;
    rec[j] = r;
  }
}

__device__ __forceinline__ bool rec_less(const SortRec& a, const SortRec& b) {
  if (a.k0 != b.k0) return a.k0 < b.k0;
  if (a.k1 != b.k1) return a.k1 < b.k1;
  if (a.seq != b.seq) return a.seq < b.seq;
  return a.row < b.row;        // NULL __seq__ first, then ties -> lower stream index (rows are numbered file by file)
}

template <class GetA, class GetB>
__device__ __forceinline__ uint32_t merge_path(uint32_t diag, uint32_t na, uint32_t nb, GetA A, GetB B) {
  uint32_t lo = diag > nb ? diag - nb : 0, hi = diag < na ? diag : na;
  while (lo < hi) {
    uint32_t mid = (lo + hi) >> 1;
    SortRec a = A(mid), b = B(diag - 1 - mid);
    if (!rec_less(b, a)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

constexpr int kMergeVT = 4;
constexpr int kMergeTile = kThreads * kMergeVT;  // 1024 records = 32 KB of shared memory

struct PairView { uint32_t a0, a1, b1; };
__device__ __forceinline__ PairView pair_of(const uint32_t* __restrict__ run_start, int k, int level, int nruns, uint32_t pos) {
  auto rstart = [&](int r) -> uint32_t { long idx = long(r) << level; return run_start[idx > k ? k : idx]; };
  int lo = 0, hi = nruns;        // upper_bound over rstart: pair containing pos = largest even r with rstart(r) <= pos
  while (lo < hi) { int mid = (lo + hi) >> 1; if (rstart(mid) <= pos) lo = mid + 1; else hi = mid; }
  int r = (lo - 1) & ~1;
  PairView p;
  p.a0 = rstart(r);
  p.a1 = rstart(r + 1 > nruns ? nruns : r + 1);
  p.b1 = rstart(r + 2 > nruns ? nruns : r + 2);
  return p;
}

// One thread per output tile: merge-path split (records taken from run A) at the tile's first output position.
// Thousands of independent binary searches overlap their latency instead of stalling every merge CTA.
__global__ void __launch_bounds__(kThreads) merge_partition_kernel(const SortRec* __restrict__ src, const uint32_t* __restrict__ run_start, int k,
                                                                  int level, const uint32_t* d_m, uint32_t* __restrict__ splits) {
  const uint32_t total = *d_m;
  const int nruns = (k + (1 << level) - 1) >> level;
  const uint32_t ntiles = (total + kMergeTile - 1) / kMergeTile;
  for (uint32_t t = blockIdx.x * kThreads + threadIdx.x; t < ntiles; t += gridDim.x * kThreads) {
    const uint32_t pos = t * kMergeTile;
    PairView p = pair_of(run_start, k, level, nruns, pos);
    const SortRec* A = src + p.a0;
    const SortRec* B = src + p.a1;
    splits[t] = merge_path(pos - p.a0, p.a1 - p.a0, p.b1 - p.a1, [&](uint32_t i) { return A[i]; }, [&](uint32_t i) { return B[i]; });
  }
}

__global__ void __launch_bounds__(kThreads) merge_pass_kernel(const SortRec* __restrict__ src, SortRec* __restrict__ dst,
                                                             const uint32_t* __restrict__ run_start, int k, int level,
                                                             const uint32_t* d_m, const uint32_t* __restrict__ splits) {
  __shared__ SortRec s_rec[kMergeTile];
  const uint32_t total = *d_m;
  const int tid = threadIdx.x;
  const int nruns = (k + (1 << level) - 1) >> level;   // runs at this level
  const uint32_t ntiles = (total + kMergeTile - 1) / kMergeTile;
  for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    uint32_t pos = tile * kMergeTile;
    const uint32_t tile_hi = pos + kMergeTile < total ? pos + kMergeTile : total;
    bool first = true;
    while (pos < tile_hi) {
      const PairView p = pair_of(run_start, k, level, nruns, pos);
      const uint32_t na = p.a1 - p.a0;
      const uint32_t seg_hi = tile_hi < p.b1 ? tile_hi : p.b1;
      const uint32_t d0 = pos - p.a0, d1 = seg_hi - p.a0;
      const SortRec* A = src + p.a0;
      const SortRec* B = src + p.a1;
      // splits: the tile's own start comes from the partition kernel; later segments start at a pair start (0);
      // a segment ends either at the pair end (na) or at the next tile's start (same pair)
      const uint32_t ia0 = first ? splits[tile] : 0u;
      const uint32_t ia1 = seg_hi == p.b1 ? na : splits[tile + 1];
      first = false;
      const uint32_t ib0 = d0 - ia0, ib1 = d1 - ia1;
      const uint32_t la = ia1 - ia0, lb = ib1 - ib0, n = la + lb;
      for (uint32_t i = tid; i < n; i += kThreads) s_rec[i] = i < la ? A[ia0 + i] : B[ib0 + (i - la)];
      __syncthreads();
      const uint32_t t0 = uint32_t(tid) * kMergeVT;
      if (t0 < n) {
        const SortRec* sA = s_rec;
        const SortRec* sB = s_rec + la;
        uint32_t ai = merge_path(t0, la, lb, [&](uint32_t i) { return sA[i]; }, [&](uint32_t i) { return sB[i]; });
        uint32_t bi = t0 - ai;
        SortRec out[kMergeVT];
        int cnt = 0;
#pragma unroll
        for (int i = 0; i < kMergeVT; i++) {
          if (t0 + i >= n) break;
          bool takeA;
          if (ai >= la) takeA = false;
          else if (bi >= lb) takeA = true;
          else takeA = !rec_less(sB[bi], sA[ai]);
          out[i] = takeA ? sA[ai++] : sB[bi++];
          cnt++;
        }
        for (int i = 0; i < cnt; i++) dst[p.a0 + d0 + t0 + i] = out[i];
      }
      __syncthreads();
      pos = seg_hi;
    }
  }
}

__global__ void __launch_bounds__(kThreads) records_to_rows_kernel(const SortRec* __restrict__ rec, const uint32_t* d_m,
                                                                  uint32_t* __restrict__ order) {
  uint32_t m = *d_m;
  for (uint32_t j = blockIdx.x * kThreads + threadIdx.x; j < m; j += gridDim.x * kThreads) order[j] = uint32_t(rec[j].row);
}

// ------------------------------------------------------------------------------------------- S5/S6: PK-run ends
// primary_key_eq (read.rs:262-287) compares VALUES only (null bitmap ignored)
__device__ __forceinline__ bool pk_equal(const PkSet& pk, uint32_t a, uint32_t b) {
  for (int c = 0; c < pk.n; c++)
    if (col_raw(pk.c[c], a) != col_raw(pk.c[c], b)) return false;
  return true;
}

__global__ void __launch_bounds__(kThreads) dedup_flags_cols_kernel(PkSet pk, const uint32_t* __restrict__ order, const uint32_t* d_m,
                                                                   uint8_t* __restrict__ keep) {
  uint32_t m = *d_m;
  for (uint32_t j = blockIdx.x * kThreads + threadIdx.x; j < m; j += gridDim.x * kThreads) {
    bool last = true;
    if (j + 1 < m) {
      uint32_t a = order ? order[j] : j, b = order ? order[j + 1] : j + 1;
      last = !pk_equal(pk, a, b);
    }
    keep[j] = last ? 1 : 0;
  }
}

__global__ void __launch_bounds__(kThreads) dedup_flags_recs_kernel(const SortRec* __restrict__ rec, const uint32_t* d_m,
                                                                   uint8_t* __restrict__ keep) {
  uint32_t m = *d_m;
  for (uint32_t j = blockIdx.x * kThreads + threadIdx.x; j < m; j += gridDim.x * kThreads) {
    bool last = true;
    if (j + 1 < m) last = rec[j].k0 != rec[j + 1].k0 || rec[j].k1 != rec[j + 1].k1;
    keep[j] = last ? 1 : 0;
  }
}

__global__ void __launch_bounds__(kThreads) gather_rows_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ out_pos,
                                                              const uint32_t* d_r, uint32_t* __restrict__ out_rows) {
  uint32_t r = *d_r;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < r; i += gridDim.x * kThreads)
    out_rows[i] = order ? order[out_pos[i]] : out_pos[i];
}

__global__ void batch_bounds_kernel(const uint32_t* __restrict__ out_pos, const uint32_t* d_r, const uint32_t* __restrict__ chunk_end,
                                    uint32_t nchunks, uint32_t* bound) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nchunks) return;
  uint32_t r = *d_r;
  uint32_t ce = chunk_end[c];
  uint32_t target = ce == 0 ? 0 : ce - 1;     // outputs with merged position < ce-1 belong to batches <= c
  uint32_t lo = 0, hi = r;
  while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (out_pos[mid] < target) lo = mid + 1; else hi = mid; }
  bound[c] = lo;
}

__global__ void chunk_ends_kernel(const uint32_t* __restrict__ surv, const uint32_t* d_m, const uint32_t* __restrict__ piece_end_row,
                                  uint32_t npieces, uint32_t* chunk_end) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= npieces) return;
  uint32_t m = *d_m, target = piece_end_row[c];
  uint32_t lo = 0, hi = m;
  if (surv == nullptr) lo = target < m ? target : m;
  else while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (surv[mid] < target) lo = mid + 1; else hi = mid; }
  chunk_end[c] = lo;
}

// ------------------------------------------------------------------------------------------- output materialisation
template <typename T>
__global__ void __launch_bounds__(kThreads) gather_column_kernel(const T* __restrict__ src, const uint8_t* __restrict__ src_valid,
                                                                const uint32_t* __restrict__ rows, const uint32_t* d_r,
                                                                T* __restrict__ dst, uint8_t* __restrict__ dst_valid) {
  uint32_t r = *d_r;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < r; i += gridDim.x * kThreads) {
    uint32_t row = rows ? rows[i] : i;
    dst[i] = src[row];
    if (dst_valid) dst_valid[i] = src_valid ? src_valid[row] : 1;
  }
}

__global__ void __launch_bounds__(kThreads) pack_validity_kernel(const uint8_t* __restrict__ valid, uint32_t n, uint8_t* __restrict__ bitmap,
                                                                unsigned long long* null_count) {
  uint32_t nbytes = (n + 7) / 8;
  uint32_t nulls = 0;
  for (uint32_t b = blockIdx.x * kThreads + threadIdx.x; b < nbytes; b += gridDim.x * kThreads) {
    uint32_t bits = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      uint32_t idx = b * 8 + i;
      if (idx < n) { if (valid[idx]) bits |= 1u << i; else nulls++; }
    }
    bitmap[b] = uint8_t(bits);
  }
  for (int d = 16; d > 0; d >>= 1) nulls += __shfl_down_sync(0xffffffffu, nulls, d);
  if ((threadIdx.x & 31) == 0 && nulls) atomicAdd(null_count, (unsigned long long)nulls);
}

// ------------------------------------------------------------------------------------------------ A1/A2: aggregation
__device__ __forceinline__ int64_t bucket_of(const AggSpecDev& s, uint32_t row) {
  int64_t ts = int64_t(widen(col_raw(s.ts, row), s.ts.type));
  return ts / s.window_ms * s.window_ms;          // truncating division == Timestamp::truncate_by (types.rs:82-85)
}

__global__ void __launch_bounds__(kThreads) group_flags_kernel(AggSpecDev spec, const uint32_t* __restrict__ rows, const uint32_t* d_r,
                                                              uint8_t* __restrict__ head) {
  uint32_t r = *d_r;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < r; i += gridDim.x * kThreads) {
    bool h = i == 0;
    if (!h) {
      uint32_t a = rows ? rows[i - 1] : i - 1, b = rows ? rows[i] : i;
      if (spec.has_group && col_raw(spec.group, a) != col_raw(spec.group, b)) h = true;
      if (!h && spec.has_ts && bucket_of(spec, a) != bucket_of(spec, b)) h = true;
    }
    head[i] = h ? 1 : 0;
  }
}

__device__ __forceinline__ double value_as_double(const ColView& c, uint32_t row) {
  uint64_t w = widen(col_raw(c, row), c.type);
  if (type_is_float(c.type)) return __longlong_as_double((long long)w);
  if (type_is_signed(c.type)) return double(int64_t(w));
  return double(w);
}

// The per-row updates of the reducers (reduce_groups_kernel, reduce_counter_groups_kernel, reduce_range_windows_kernel): one thread
// takes a group's non-NULL values in stream order, each converted to f64.
// sum / min / max: the f64 sum is a strictly sequential chain (SURVEY §8a A2); min / max start at +inf / -inf
struct SumMinMax { double sum, mn, mx; bool seen; };
__device__ __forceinline__ SumMinMax sum_min_max_init() {
  return SumMinMax{0.0, __longlong_as_double(0x7ff0000000000000LL), __longlong_as_double((long long)0xfff0000000000000ULL), false};
}
__device__ __forceinline__ void sum_min_max_add(SumMinMax& a, double v) {
  a.sum += v;
  if (!a.seen || v < a.mn) a.mn = v;
  if (!a.seen || v > a.mx) a.mx = v;
  a.seen = true;
}

// Counter partials over v1..vm: resets = #{i >= 2 : v_i < v_(i-1)}, increase = sequential f64 sum of (v_i < v_(i-1) ? v_i : v_i - v_(i-1))
// (a drop is a counter restart from 0; a comparison with a NaN is false, so never a reset).  first / last: the position (a row id, or an
// index) of the first / last value, whose time the caller reads.  prev ends as the last value.
struct CounterAcc { double first_v, prev, inc; uint64_t resets; uint32_t first, last; bool seen; };
__device__ __forceinline__ CounterAcc counter_init() { return CounterAcc{0.0, 0.0, 0.0, 0, 0, 0, false}; }
__device__ __forceinline__ void counter_add(CounterAcc& c, double v, uint32_t at) {
  if (!c.seen) {
    c.first_v = v;
    c.first = at;
    c.seen = true;
  } else if (v < c.prev) {
    c.inc += v;
    c.resets++;
  } else {
    c.inc += v - c.prev;
  }
  c.prev = v;
  c.last = at;
}

// one rounding per operation: nvcc would contract `a * b + c` into an FMA (host compilers of the emulated build do not)
__device__ __forceinline__ double mul_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__device__ __forceinline__ double add_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

// One thread per group walks its rows in stream order.
__global__ void __launch_bounds__(kThreads) reduce_groups_kernel(AggSpecDev spec, const uint32_t* __restrict__ rows, const uint32_t* d_r,
                                                                const uint32_t* __restrict__ seg_start, const uint32_t* d_g, AggOut out) {
  uint32_t g_total = *d_g, r_total = *d_r;
  for (uint32_t g = blockIdx.x * kThreads + threadIdx.x; g < g_total; g += gridDim.x * kThreads) {
    uint32_t lo = seg_start[g], hi = g + 1 < g_total ? seg_start[g + 1] : r_total;
    uint32_t first = rows ? rows[lo] : lo;
    if (out.gkey) {
      uint64_t kv = spec.has_group ? col_raw(spec.group, first) : 0;
      store_val_dyn(out.gkey, spec.has_group ? spec.group.width : 8, g, kv);
    }
    out.bucket[g] = spec.has_ts ? bucket_of(spec, first) : 0;
    out.count[g] = hi - lo;
    SumMinMax a = sum_min_max_init();
    if (spec.has_value) {
      for (uint32_t i = lo; i < hi; i++) {
        uint32_t row = rows ? rows[i] : i;
        if (!col_valid(spec.value, row)) continue;
        sum_min_max_add(a, value_as_double(spec.value, row));
      }
    }
    out.sum[g] = a.sum;
    out.min[g] = a.mn;
    out.max[g] = a.mx;
  }
}

// Counter partials: one thread per group walks its rows in stream order, like reduce_groups.  The time column is read for the first and
// last valid rows only.
__global__ void __launch_bounds__(kThreads) reduce_counter_groups_kernel(AggSpecDev spec, const uint32_t* __restrict__ rows, const uint32_t* d_r,
                                                                        const uint32_t* __restrict__ seg_start, const uint32_t* d_g, CounterOut out) {
  uint32_t g_total = *d_g, r_total = *d_r;
  for (uint32_t g = blockIdx.x * kThreads + threadIdx.x; g < g_total; g += gridDim.x * kThreads) {
    uint32_t lo = seg_start[g], hi = g + 1 < g_total ? seg_start[g + 1] : r_total;
    uint32_t first = rows ? rows[lo] : lo;
    store_val_dyn(out.gkey, spec.group.width, g, col_raw(spec.group, first));
    out.bucket[g] = spec.has_ts ? bucket_of(spec, first) : 0;
    out.count[g] = hi - lo;
    CounterAcc c = counter_init();
    for (uint32_t i = lo; i < hi; i++) {
      uint32_t row = rows ? rows[i] : i;
      if (!col_valid(spec.value, row)) continue;
      counter_add(c, value_as_double(spec.value, row), row);
    }
    out.first_ts[g] = c.seen ? int64_t(widen(col_raw(spec.ts, c.first), spec.ts.type)) : 0;
    out.first_value[g] = c.first_v;
    out.last_ts[g] = c.seen ? int64_t(widen(col_raw(spec.ts, c.last), spec.ts.type)) : 0;
    out.last_value[g] = c.prev;
    out.increase[g] = c.inc;
    out.resets[g] = c.resets;
    out.valid[g] = c.seen ? 1 : 0;
  }
}

// ------------------------------------------------------------------------------------------------ range windows (hg_scan_range_aggregate)
// Input: the groups of group_rows, one per series: agg row t -> decoded row rows[t], series g = agg rows [seg[g], seg[g+1]), head[t] = 1 on
// a series' first row.  Every row passed the call's time bounds (start - range < ts <= end).
//   gather    ts (widened to i64), value (f64) and validity in agg-row order: the windows read these contiguous arrays
//   count     row t lies in the windows [lo_t, hi_t] (range_steps) and opens those of them past its predecessor's: [max(lo_t, hi_(t-1) + 1),
//             hi_t]; per block of kRangeTile rows the windows opened and the row memberships (u64), then one block scans the block sums
//   windows   after the host read the window count: the exclusive scan of the per-row counts (each window's slot), then one thread per
//             window finds the row that opens it (binary search in the scan) and its end (the first row of the series past t_j)
//   reduce    one thread per window walks its rows in stream order: ten columns in one pass
constexpr int kRangePerThread = 8;
constexpr uint32_t kRangeTile = kThreads * kRangePerThread;

struct RangeSteps { int64_t lo, hi; };
// the windows j holding time ts: t_j in [ts, ts + range - 1], i.e. lo = max(0, ceil((ts - start) / step)), hi = min(n - 1, floor((ts + range
// - 1 - start) / step)); lo > hi: none.  Within the time bounds ts - start and ts + range - 1 - start fit in i64 (the host's checks), and
// the second is >= 0.
__device__ __forceinline__ RangeSteps range_steps(const RangeSpecDev& r, int64_t ts) {
  const int64_t d = ts - r.start, e = d + (r.range - 1);
  RangeSteps s;
  s.lo = d <= 0 ? 0 : d / r.step + (d % r.step != 0);
  s.hi = e < 0 ? -1 : e / r.step;
  if (s.hi > int64_t(r.n) - 1) s.hi = int64_t(r.n) - 1;
  return s;
}

// the first window row t opens (it opens [first, s.hi]): windows up to its predecessor's last one already have a first row
__device__ __forceinline__ int64_t range_first_open(const RangeSpecDev& r, const int64_t* ts, const uint8_t* head, uint32_t t, RangeSteps s) {
  if (!head[t]) {
    const int64_t after_prev = range_steps(r, ts[t - 1]).hi + 1;
    if (after_prev > s.lo) return after_prev;
  }
  return s.lo;
}

__global__ void __launch_bounds__(kThreads) range_gather_kernel(ColView ts, ColView value, const uint32_t* __restrict__ rows, const uint32_t* d_r,
                                                               int64_t* __restrict__ ts_out, double* __restrict__ v_out, uint8_t* __restrict__ ok_out) {
  const uint32_t r = *d_r;
  for (uint32_t t = blockIdx.x * kThreads + threadIdx.x; t < r; t += gridDim.x * kThreads) {
    const uint32_t row = rows ? rows[t] : t;
    const bool ok = col_valid(value, row);
    ts_out[t] = int64_t(widen(col_raw(ts, row), ts.type));
    v_out[t] = ok ? value_as_double(value, row) : 0.0;
    ok_out[t] = ok ? 1 : 0;
  }
}

// cnt[t] = the windows row t opens; per block b: wsum[b] = their sum, msum[b] = the rows' window memberships (sum of hi_t - lo_t + 1)
__global__ void __launch_bounds__(kThreads) range_count_kernel(RangeSpecDev rs, const int64_t* __restrict__ ts, const uint8_t* __restrict__ head,
                                                              const uint32_t* d_r, uint32_t* __restrict__ cnt, uint64_t* __restrict__ wsum,
                                                              uint64_t* __restrict__ msum) {
  __shared__ uint64_t s_w64[9];
  const uint32_t r = *d_r, nb = (r + kRangeTile - 1) / kRangeTile;
  for (uint32_t b = blockIdx.x; b < nb; b += gridDim.x) {
    uint64_t opened = 0, members = 0;
    const uint32_t base = b * kRangeTile + threadIdx.x * kRangePerThread;
    for (uint32_t i = 0; i < kRangePerThread && base + i < r; i++) {
      const uint32_t t = base + i;
      const RangeSteps s = range_steps(rs, ts[t]);
      const int64_t first = range_first_open(rs, ts, head, t, s);
      const uint32_t c = s.hi >= first ? uint32_t(s.hi - first + 1) : 0u;
      cnt[t] = c;
      opened += c;
      if (s.hi >= s.lo) members += uint64_t(s.hi - s.lo + 1);
    }
    uint64_t total_opened, total_members;
    (void)block_incl_scan64(opened, &total_opened, s_w64);
    (void)block_incl_scan64(members, &total_members, s_w64);
    if (threadIdx.x == 0) {
      wsum[b] = total_opened;
      msum[b] = total_members;
    }
  }
}

// one block: wsum becomes its exclusive scan; totals[0] = the windows, totals[1] = the memberships (the sum of the window lengths)
__global__ void __launch_bounds__(kThreads) range_scan_sums_kernel(uint64_t* wsum, const uint64_t* __restrict__ msum, const uint32_t* d_r,
                                                                  uint64_t* totals) {
  __shared__ uint64_t s_w64[9];
  const uint32_t r = *d_r, nb = (r + kRangeTile - 1) / kRangeTile;
  uint64_t carry = 0, members = 0;
  for (uint32_t base = 0; base < nb; base += kThreads) {
    const uint32_t i = base + threadIdx.x;
    const uint64_t v = i < nb ? wsum[i] : 0;
    uint64_t total, total_m;
    const uint64_t inc = block_incl_scan64(v, &total, s_w64);
    if (i < nb) wsum[i] = carry + inc - v;
    carry += total;
    (void)block_incl_scan64(i < nb ? msum[i] : 0, &total_m, s_w64);
    members += total_m;
  }
  if (threadIdx.x == 0) {
    totals[0] = carry;
    totals[1] = members;
  }
}

// cnt[t] -> its exclusive scan (the slot of the first window row t opens); the host has checked that the window count fits in u32
__global__ void __launch_bounds__(kThreads) range_offsets_kernel(const uint64_t* __restrict__ wsum, const uint32_t* d_r, uint32_t* __restrict__ cnt) {
  __shared__ uint32_t s_warp[9];
  const uint32_t r = *d_r, nb = (r + kRangeTile - 1) / kRangeTile;
  for (uint32_t b = blockIdx.x; b < nb; b += gridDim.x) {
    const uint32_t base = b * kRangeTile + threadIdx.x * kRangePerThread;
    uint32_t c[kRangePerThread], sum = 0;
#pragma unroll
    for (int i = 0; i < kRangePerThread; i++) {
      c[i] = base + i < r ? cnt[base + i] : 0u;
      sum += c[i];
    }
    uint32_t total;
    uint32_t o = uint32_t(wsum[b]) + block_excl_scan<kThreads>(sum, &total, s_warp);
#pragma unroll
    for (int i = 0; i < kRangePerThread; i++)
      if (base + i < r) {
        cnt[base + i] = o;
        o += c[i];
      }
  }
}

// One thread per window w: the row t that opens it is the last one with off[t] <= w, its step j = range_first_open + (w - off[t]); the
// window is agg rows [t, end) with end = the first row of t's series with ts > t_j.  *members = the sum of the window lengths.
__global__ void __launch_bounds__(kThreads) range_windows_kernel(RangeSpecDev rs, const int64_t* __restrict__ ts, const uint8_t* __restrict__ head,
                                                                const uint32_t* __restrict__ off, const uint32_t* d_r, const uint32_t* __restrict__ seg,
                                                                uint32_t G, ColView group, const uint32_t* __restrict__ rows, uint32_t W,
                                                                RangeWindows out) {
  const uint32_t r = *d_r;
  for (uint32_t w = blockIdx.x * kThreads + threadIdx.x; w < W; w += gridDim.x * kThreads) {
    uint32_t a = 0, b = r;
    while (a < b) { const uint32_t h = a + ((b - a) >> 1); if (off[h] <= w) a = h + 1; else b = h; }
    const uint32_t t = a - 1;
    const int64_t tj = rs.start + (range_first_open(rs, ts, head, t, range_steps(rs, ts[t])) + int64_t(w - off[t])) * rs.step;
    uint32_t ga = 0, gb = G;                                // t's series ends at the first series start past t
    while (ga < gb) { const uint32_t h = ga + ((gb - ga) >> 1); if (seg[h] <= t) ga = h + 1; else gb = h; }
    uint32_t ka = t + 1, kb = ga < G ? seg[ga] : r;
    while (ka < kb) { const uint32_t h = ka + ((kb - ka) >> 1); if (ts[h] <= tj) ka = h + 1; else kb = h; }
    out.lo[w] = t;
    out.hi[w] = ka;
    out.t[w] = tj;
    store_val_dyn(out.gkey, group.width, w, col_raw(group, rows ? rows[t] : t));
  }
}

// One thread per window walks its rows [lo, hi) of the gathered arrays in stream order: count, sum / min / max and the counter partials
__global__ void __launch_bounds__(kThreads) reduce_range_windows_kernel(const int64_t* __restrict__ ts, const double* __restrict__ v,
                                                                       const uint8_t* __restrict__ ok, const uint32_t* __restrict__ win_lo,
                                                                       const uint32_t* __restrict__ win_hi, uint32_t W, RangeOut out) {
  for (uint32_t w = blockIdx.x * kThreads + threadIdx.x; w < W; w += gridDim.x * kThreads) {
    const uint32_t lo = win_lo[w], hi = win_hi[w];
    SumMinMax a = sum_min_max_init();
    CounterAcc c = counter_init();
    for (uint32_t i = lo; i < hi; i++) {
      if (!ok[i]) continue;
      const double x = v[i];
      sum_min_max_add(a, x);
      counter_add(c, x, i);
    }
    out.count[w] = hi - lo;
    out.sum[w] = a.sum;
    out.min[w] = a.mn;
    out.max[w] = a.mx;
    out.first_ts[w] = c.seen ? ts[c.first] : 0;
    out.first_value[w] = c.first_v;
    out.last_ts[w] = c.seen ? ts[c.last] : 0;
    out.last_value[w] = c.prev;
    out.increase[w] = c.inc;
    out.resets[w] = c.resets;
    out.valid[w] = c.seen ? 1 : 0;
  }
}

// ------------------------------------------------------------------------------------------ range functions (hg_scan_range_function)
// One thread per window over the gathered arrays of range_count: the window's samples are its rows with ok[i], in stream order,
// (T_0, V_0) .. (T_(m-1), V_(m-1)).  The definitions are include/horae_gpu.h's, every f64 operation rounded on its own (mul_rn / add_rn,
// plain IEEE division): a contracted FMA would change the last bit.  Returns false when the window has no value.
__device__ __forceinline__ bool range_fn_value(const RangeFnSpec& f, const int64_t* __restrict__ ts, const double* __restrict__ v,
                                               const uint8_t* __restrict__ ok, uint32_t lo, uint32_t hi, int64_t t, double* out) {
  uint32_t last = hi;                                 // one past the last sample: a short scan back from the window's end
  while (last > lo && !ok[last - 1]) last--;
  if (last == lo) return false;                       // m = 0
  const uint32_t il = last - 1;
  if (f.fn == kFnIrate || f.fn == kFnIdelta) {
    uint32_t prev = il;                               // one past the second-to-last sample
    while (prev > lo && !ok[prev - 1]) prev--;
    if (prev == lo) return false;
    const uint32_t ia = prev - 1;
    if (ts[il] == ts[ia]) return false;
    const double va = v[ia], vb = v[il];
    if (f.fn == kFnIdelta) { *out = add_rn(vb, -va); return true; }
    *out = (vb < va ? vb : add_rn(vb, -va)) / (double(ts[il] - ts[ia]) / 1000.0);
    return true;
  }
  uint32_t i0 = lo;
  while (!ok[i0]) i0++;                               // the first sample (il is one)
  const double v0 = v[i0];
  if (f.fn <= kFnDelta) {
    if (i0 == il || ts[i0] == ts[il]) return false;   // m = 1, or every sample at one time
    const bool counter = f.fn != kFnDelta;
    double result = add_rn(v[il], -v0), prev = v0;
    uint32_t m = 1;
    for (uint32_t i = i0 + 1; i <= il; i++) {
      if (!ok[i]) continue;
      const double x = v[i];
      if (counter && x < prev) result = add_rn(result, prev);
      prev = x;
      m++;
    }
    double d_start = double(ts[i0] - (t - f.range)) / 1000.0;
    double d_end = double(t - ts[il]) / 1000.0;
    const double sampled = double(ts[il] - ts[i0]) / 1000.0;
    const double avg = sampled / double(m - 1);
    const double thr = mul_rn(avg, 1.1);
    if (d_start >= thr) d_start = avg / 2.0;
    if (counter && result > 0.0 && v0 >= 0.0) {
      const double d_zero = mul_rn(sampled, v0 / result);
      if (d_zero < d_start) d_start = d_zero;
    }
    double ext = add_rn(sampled, d_start);
    if (d_end >= thr) d_end = avg / 2.0;
    ext = add_rn(ext, d_end);
    double factor = ext / sampled;
    if (f.fn == kFnRate) factor = factor / f.range_s;
    *out = mul_rn(result, factor);
    return true;
  }
  if (f.fn == kFnLastOverTime) { *out = v[il]; return true; }
  // one forward pass: resets, changes, count / sum / min / max over time
  SumMinMax a = sum_min_max_init();
  uint64_t resets = 0, changes = 0, m = 0;
  double prev = v0;
  for (uint32_t i = i0; i <= il; i++) {
    if (!ok[i]) continue;
    const double x = v[i];
    if (m) {
      if (x < prev) resets++;
      if (!(x == prev || (x != x && prev != prev))) changes++;
    }
    sum_min_max_add(a, x);
    prev = x;
    m++;
  }
  switch (f.fn) {
    case kFnResets: *out = double(resets); break;
    case kFnChanges: *out = double(changes); break;
    case kFnCountOverTime: *out = double(m); break;
    case kFnSumOverTime: *out = a.sum; break;
    case kFnMinOverTime: *out = a.mn; break;
    default: *out = a.mx; break;                      // kFnMaxOverTime (the host checked fn)
  }
  return true;
}

__global__ void __launch_bounds__(kThreads) range_function_kernel(RangeFnSpec f, const int64_t* __restrict__ ts, const double* __restrict__ v,
                                                                 const uint8_t* __restrict__ ok, const uint32_t* __restrict__ win_lo,
                                                                 const uint32_t* __restrict__ win_hi, const int64_t* __restrict__ win_t, uint32_t W,
                                                                 double* __restrict__ value, uint8_t* __restrict__ valid) {
  for (uint32_t w = blockIdx.x * kThreads + threadIdx.x; w < W; w += gridDim.x * kThreads) {
    double x = 0.0;
    const bool has = range_fn_value(f, ts, v, ok, win_lo[w], win_hi[w], win_t[w], &x);
    value[w] = x;
    valid[w] = has ? 1 : 0;
  }
}

// The windows with a value, idx[0 .. *d_n) in (series, t) order, gathered into the per-series result
__global__ void __launch_bounds__(kThreads) range_fn_gather_kernel(const uint32_t* __restrict__ idx, const uint32_t* d_n, ColView key,
                                                                  const int64_t* __restrict__ t, const double* __restrict__ value, void* key_out,
                                                                  int64_t* __restrict__ t_out, double* __restrict__ value_out) {
  const uint32_t n = *d_n;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    const uint32_t w = idx[i];
    store_val_dyn(key_out, key.width, i, col_raw(key, w));
    t_out[i] = t[w];
    value_out[i] = value[w];
  }
}

// The sort keys of the by-map result: (ordinal << shift) | j with j = the window's step, vals = the window
__global__ void __launch_bounds__(kThreads) range_fn_sort_keys_kernel(const uint32_t* __restrict__ idx, const uint32_t* d_n,
                                                                     const uint32_t* __restrict__ ordinal, const int64_t* __restrict__ t,
                                                                     int64_t start, int64_t step, int shift, uint64_t* __restrict__ keys,
                                                                     uint32_t* __restrict__ vals) {
  const uint32_t n = *d_n;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    const uint32_t w = idx[i];
    keys[i] = (uint64_t(ordinal[w]) << shift) | uint64_t((t[w] - start) / step);
    vals[i] = w;
  }
}

// ------------------------------------------------------------------------------ top-k / bottom-k per group (hg_scan_range_function_topk)
// The rank key of window idx[i]'s value: ascending in the result's order, -0.0 taken as +0.0, every NaN the largest key (last in both
// directions).  f64_total_order_key of the canonical bits, complemented for the descending order; integer operations only.
__global__ void __launch_bounds__(kThreads) topk_rank_keys_kernel(const uint32_t* __restrict__ idx, const uint32_t* d_n,
                                                                 const double* __restrict__ value, int descending, uint64_t* __restrict__ keys) {
  const uint32_t n = *d_n;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    const uint64_t b = uint64_t(__double_as_longlong(value[idx[i]]));
    const uint64_t mag = b & 0x7fffffffffffffffull;
    uint64_t key = ~0ull;
    if (mag <= 0x7ff0000000000000ull) {
      key = f64_total_order_key(mag ? b : 0ull);
      if (descending) key = ~key;                  // at least 0xfff0000000000000 (-inf) below the NaN key
    }
    keys[i] = key;
  }
}

// keep[i] = window i of the sorted windows is among the first k of its segment (segments: seg[0 .. d_n[1]), windows: [0, d_n[0])); 0 from
// d_n[0] to cap
__global__ void __launch_bounds__(kThreads) topk_keep_kernel(const uint32_t* __restrict__ seg, const uint32_t* d_n, uint32_t cap, uint32_t k,
                                                            uint8_t* __restrict__ keep) {
  const uint32_t n = d_n[0], S = d_n[1];
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < cap; i += gridDim.x * kThreads) {
    uint8_t f = 0;
    if (i < n) {
      uint32_t a = 0, b = S;                       // the last segment that starts at or before i (seg[0] == 0)
      while (a < b) { const uint32_t h = a + ((b - a) >> 1); if (seg[h] <= i) a = h + 1; else b = h; }
      f = i - seg[a - 1] < k ? 1 : 0;
    }
    keep[i] = f;
  }
}

// The kept windows win[pos[0 .. *d_r)] gathered into the result: the ordinal, t, the series key (the key column at the row that opens the
// window, agg row win_lo[w] -> decoded row rows[..]) and the value with its bits
__global__ void __launch_bounds__(kThreads) topk_gather_kernel(const uint32_t* __restrict__ pos, const uint32_t* d_r, const uint32_t* __restrict__ win,
                                                              const uint32_t* __restrict__ ordinal, const int64_t* __restrict__ t,
                                                              const double* __restrict__ value, const uint32_t* __restrict__ win_lo, ColView series,
                                                              const uint32_t* __restrict__ rows, TopkOut out) {
  const uint32_t r = *d_r;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < r; i += gridDim.x * kThreads) {
    const uint32_t w = win[pos[i]], lo = win_lo[w];
    out.group[i] = ordinal[w];
    out.t[i] = t[w];
    store_val_dyn(out.key, series.width, i, col_raw(series, rows ? rows[lo] : lo));
    out.value[i] = value[w];
  }
}

// ------------------------------------------------------------------------------------ histogram quantiles (hg_scan_histogram_quantile)
// The sort keys of the bucket sums: (group rank, step, bound rank), so that one (group, t)'s buckets are adjacent in bound order
__global__ void __launch_bounds__(kThreads) histogram_sort_keys_kernel(const uint32_t* __restrict__ idx, const uint32_t* d_n,
                                                                      const uint32_t* __restrict__ ordinal, const BucketPair* __restrict__ pair,
                                                                      const int64_t* __restrict__ t, int64_t start, int64_t step, int shift,
                                                                      int lbits, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const uint32_t n = *d_n;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    const uint32_t w = idx[i];
    const BucketPair p = pair[ordinal[w]];
    keys[i] = (uint64_t(p.group) << (shift + lbits)) | (uint64_t((t[w] - start) / step) << lbits) | uint64_t(p.bound);
    vals[i] = w;
  }
}

__global__ void __launch_bounds__(kThreads) histogram_heads_kernel(const uint32_t* __restrict__ ordinal, const int64_t* __restrict__ t,
                                                                  const BucketPair* __restrict__ pair, const uint32_t* d_n, uint8_t* __restrict__ head) {
  const uint32_t n = *d_n;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads)
    head[i] = (i == 0 || t[i] != t[i - 1] || pair[ordinal[i]].group != pair[ordinal[i - 1]].group) ? 1 : 0;
}

// util/almost.Equal(a, b, 1e-12) of Prometheus: relative difference below 1e-12, absolute below 1e-12 * 2^-1022 near zero
__device__ __forceinline__ bool almost_equal(double a, double b) {
  if ((a != a && b != b) || a == b) return true;
  const double s = add_rn(fabs(a), fabs(b)), d = fabs(add_rn(a, -b));
  const double min_normal = __longlong_as_double(0x0010000000000000LL);          // 2^-1022
  if (a == 0.0 || b == 0.0 || s < min_normal) return d < __longlong_as_double(0x1198LL);   // the f64 product 1e-12 * 2^-1022 (subnormal)
  const double max_f64 = __longlong_as_double(0x7fefffffffffffffLL);
  return d / (s != s || s < max_f64 ? s : max_f64) < 1e-12;                     // Go's math.Min: NaN stays NaN
}

// bucketQuantile's steps 5-7 (include/horae_gpu.h) over n >= 2 fixed-up counts c[0 .. n) with obs = c[n - 1] != 0: sort.Search's binary
// search for the first bucket with c >= rank among the first n - 1, then the linear interpolation inside it
template <typename Upper>
__device__ __forceinline__ double bucket_quantile(double q, const double* c, uint32_t n, const Upper& upper) {
  double rank = mul_rn(q, c[n - 1]);
  uint32_t lo = 0, hi = n - 1;
  while (lo < hi) {
    const uint32_t h = (lo + hi) >> 1;
    if (!(c[h] >= rank)) lo = h + 1;
    else hi = h;
  }
  const uint32_t b = lo;
  if (b == n - 1) return upper(n - 2);
  const double end = upper(b);
  if (b == 0 && end <= 0.0) return end;
  double start = 0.0, cnt = c[b];
  if (b > 0) {
    start = upper(b - 1);
    cnt = add_rn(cnt, -c[b - 1]);
    rank = add_rn(rank, -c[b - 1]);
  }
  return add_rn(start, mul_rn(add_rn(end, -start), rank / cnt));
}

// One thread per (group, t) segment of bucket sums in bound order: steps 1-7 of include/horae_gpu.h for every q.  The fix-up runs once
// and writes the counts in place, so that every q's binary search sees the fixed counts.
__global__ void __launch_bounds__(kThreads) histogram_quantile_kernel(QuantileSpec qs, const uint32_t* __restrict__ seg, uint32_t S, uint32_t rows,
                                                                     const uint32_t* __restrict__ ordinal, const int64_t* __restrict__ t,
                                                                     double* __restrict__ count, const BucketPair* __restrict__ pair,
                                                                     const double* __restrict__ bounds, const uint32_t* __restrict__ group_ordinal,
                                                                     HistogramOut out) {
  const double inf = __longlong_as_double(0x7ff0000000000000LL), nan = __longlong_as_double(0x7ff8000000000000LL);
  for (uint32_t s = blockIdx.x * kThreads + threadIdx.x; s < S; s += gridDim.x * kThreads) {
    const uint32_t lo = seg[s], n = (s + 1 < S ? seg[s + 1] : rows) - lo;
    double* c = count + lo;
    auto upper = [&](uint32_t i) { return bounds[pair[ordinal[lo + i]].bound]; };
    out.group[s] = group_ordinal[pair[ordinal[lo]].group];
    out.t[s] = t[lo];
    bool forced = false, none = !(upper(n - 1) == inf);             // 1: no +inf bucket
    if (!none) {
      double prev = c[0];                                            // 3: the fix-up
      for (uint32_t i = 1; i < n; i++) {
        const double cur = c[i];
        if (cur == prev) continue;
        if (almost_equal(prev, cur)) { c[i] = prev; continue; }
        if (cur < prev) { c[i] = prev; forced = true; continue; }
        prev = cur;
      }
      none = n < 2 || c[n - 1] == 0.0;                               // 4
    }
    out.forced[s] = forced ? 1 : 0;
    for (uint32_t j = 0; j < qs.n; j++) out.q[size_t(j) * S + s] = none ? nan : bucket_quantile(qs.q[j], c, n, upper);
  }
}

__global__ void pack_agg_kernel(AggOut in, uint32_t gwidth, uint64_t g, uint64_t cap, long long* __restrict__ dst) {
  for (uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < cap; i += uint64_t(gridDim.x) * blockDim.x) {
    const bool v = i < g;
    long long key = 0;
    if (v) {
      switch (gwidth) {
        case 1: key = reinterpret_cast<const uint8_t*>(in.gkey)[i]; break;
        case 2: key = reinterpret_cast<const uint16_t*>(in.gkey)[i]; break;
        case 4: key = reinterpret_cast<const uint32_t*>(in.gkey)[i]; break;
        default: key = (long long)reinterpret_cast<const uint64_t*>(in.gkey)[i];
      }
    }
    dst[i] = key;
    dst[cap + i] = v ? in.bucket[i] : 0;
    dst[2 * cap + i] = v ? (long long)in.count[i] : 0;
    dst[3 * cap + i] = v ? __double_as_longlong(in.sum[i]) : 0;
    dst[4 * cap + i] = v ? __double_as_longlong(in.min[i]) : 0;
    dst[5 * cap + i] = v ? __double_as_longlong(in.max[i]) : 0;
  }
}

// ------------------------------------------------------------------------------------------- Binary columns: export
// byte length of the i-th output row (0 for NULL and beyond the count), for an exclusive scan -> Arrow offsets
__global__ void __launch_bounds__(kThreads) gather_lens_kernel(ColView col, const uint32_t* __restrict__ rows, const uint32_t* d_n, uint32_t cap,
                                                              uint32_t* __restrict__ out) {
  const uint32_t n = *d_n;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < cap; i += gridDim.x * kThreads) {
    uint32_t len = 0;
    if (i < n) { const uint32_t row = rows ? rows[i] : i; if (col.valid == nullptr || col.valid[row]) len = col.lens[row]; }
    out[i] = len;
  }
}
// one warp per row: bytes of row rows[i] -> dst + offs[i]
__global__ void __launch_bounds__(kThreads) copy_var_kernel(ColView col, const uint32_t* __restrict__ rows, const uint32_t* d_n,
                                                           const uint32_t* __restrict__ offs, uint8_t* __restrict__ dst) {
  const uint32_t n = *d_n;
  const int lane = threadIdx.x & 31;
  const uint32_t nwarps = gridDim.x * (kThreads / 32);
  for (uint32_t i = (blockIdx.x * kThreads + threadIdx.x) >> 5; i < n; i += nwarps) {
    const uint32_t row = rows ? rows[i] : i;
    if (col.valid && !col.valid[row]) continue;
    const uint8_t* src = reinterpret_cast<const uint8_t* const*>(col.vals)[row];
    const uint32_t len = col.lens[row];
    uint8_t* d = dst + offs[i];
    for (uint32_t b = lane; b < len; b += 32) d[b] = src[b];
  }
}
// Append mode: first row of the j-th primary-key run in merged order (the run ends at merged position out_pos[j])
__global__ void __launch_bounds__(kThreads) first_rows_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ out_pos, const uint32_t* d_r,
                                                             uint32_t* __restrict__ out) {
  const uint32_t r = *d_r;
  for (uint32_t j = blockIdx.x * kThreads + threadIdx.x; j < r; j += gridDim.x * kThreads) {
    const uint32_t pos = j ? out_pos[j - 1] + 1 : 0;
    out[j] = order ? order[pos] : pos;
  }
}
// Append mode: Arrow offsets of the concatenated values = the running byte count sampled at the runs' first rows (+ the total)
__global__ void __launch_bounds__(kThreads) run_offsets_kernel(const uint32_t* __restrict__ cum, const uint32_t* __restrict__ out_pos, const uint32_t* d_r,
                                                              const uint32_t* d_m, uint32_t* __restrict__ out) {
  const uint32_t r = *d_r, m = *d_m;
  for (uint32_t j = blockIdx.x * kThreads + threadIdx.x; j <= r; j += gridDim.x * kThreads)
    out[j] = j == r ? cum[m] : cum[j ? out_pos[j - 1] + 1 : 0];
}

__global__ void __launch_bounds__(kThreads) append_validity_kernel(ColView col, const uint32_t* __restrict__ order, const uint32_t* __restrict__ out_pos,
                                                                  const uint32_t* d_r, const uint32_t* __restrict__ run_offs, uint8_t* __restrict__ valid, int* err) {
  const uint32_t r = *d_r;
  for (uint32_t j = blockIdx.x * kThreads + threadIdx.x; j < r; j += gridDim.x * kThreads) {
    uint8_t v = 1;
    if (run_offs[j + 1] == run_offs[j]) {
      const uint32_t first = j ? out_pos[j - 1] + 1 : 0, last = out_pos[j];
      if (first == last) { const uint32_t row = order ? order[first] : first; v = (col.valid == nullptr || col.valid[row]) ? 1 : 0; }
      else atomicExch(err, 130);
    }
    valid[j] = v;
  }
}

__global__ void fill_u32_kernel(uint32_t* p, uint32_t v, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = v;
}

__global__ void uniform_chunk_ends_kernel(const uint32_t* d_m, uint32_t batch, uint32_t nchunks, uint32_t* chunk_end) {
  uint32_t m = *d_m;
  for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += gridDim.x * blockDim.x) {
    uint64_t e = uint64_t(c + 1) * batch;
    chunk_end[c] = e < m ? uint32_t(e) : m;
  }
}
__global__ void clear_tail_kernel(uint8_t* flags, const uint32_t* d_n, uint32_t cap) {
  uint32_t n = *d_n;
  for (uint64_t i = uint64_t(n) + blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += uint64_t(gridDim.x) * blockDim.x) flags[i] = 0;
}

// ------------------------------------------------------------------------------------------------ A2: quantiles per group
// Exact quantiles per group (hg_scan_quantile_aggregate).
// Input: the general pipeline's groups (engine.cu: group_rows): agg row t -> decoded row rows[t], group g = agg rows [seg[g], seg[g+1]).
//   prepare   value flags, compaction of the non-NULL rows (compact_flags), their order keys in group order, then one thread per group:
//             its slice [start, start + m) of the keys, the NULL result of an empty group, and its tier (one small D2H sizes the rest)
//   small     m <= kQuantileSmallMax: one warp per group, a bitonic network over 64-bit keys in registers (shuffles)
//   medium    m <= kQuantileMediumMax: one block per group, a bitonic sort in shared memory
//   large     radix select: 8 passes of 8-bit digits from the top, every pending rank of a group in the same pass with its own prefix and
//             256-bin histogram.  A pass is one histogram launch, a block per chunk of kQuantileChunk keys (a group above that is spread
//             over many blocks, global histograms with atomics), and one resolve launch (one warp per group picks each rank's digit).
//             This tier reads its keys once per pass: 8 times.
// Every tier converts the selected keys back to values (order_key_to_plain, widen, then f64) and interpolates with mul_rn / add_rn
// (__dmul_rn / __dadd_rn on the device), so that no multiply-add is contracted into an FMA: the result is the formula of
// include/horae_gpu.h, rounded step by step.

constexpr uint32_t kRanks = 2 * kQuantileMax;    // the distinct ranks lo / hi a group of the large tier may need
constexpr uint32_t kFull = 0xffffffffu;

// the value of an order key (order_key(widen(x))) as an f64: integers above 2^53 round to nearest
__device__ __forceinline__ double key_value(uint64_t key, uint32_t type) {
  const uint64_t w = widen(order_key_to_plain(key, type), type);
  if (type_is_float(type)) return __longlong_as_double((long long)w);
  return type_is_signed(type) ? double(int64_t(w)) : double(w);
}

struct QRank { uint32_t lo, hi; double w; };
// rank = q * (m - 1), lo = floor(rank), hi = min(lo + 1, m - 1), w = rank - lo   (m >= 1)
__device__ __forceinline__ QRank quantile_rank(double q, uint32_t m) {
  const double rank = mul_rn(q, double(m - 1));
  const double f = floor(rank);
  const uint32_t lo = uint32_t(f);
  return QRank{lo, lo + 1 < m ? lo + 1 : m - 1, rank - f};
}

__device__ __forceinline__ double interpolate(uint64_t klo, uint64_t khi, double w, uint32_t type) {
  const double a = key_value(klo, type);
  if (w == 0.0) return a;
  return add_rn(mul_rn(a, 1.0 - w), mul_rn(key_value(khi, type), w));
}

__global__ void __launch_bounds__(kThreads) quantile_flags_kernel(ColView value, const uint32_t* __restrict__ rows, const uint32_t* d_r,
                                                                   uint32_t cap, uint8_t* __restrict__ flags) {
  const uint32_t r = *d_r;
  for (uint32_t t = blockIdx.x * kThreads + threadIdx.x; t < cap; t += gridDim.x * kThreads)
    flags[t] = t < r && col_valid(value, rows ? rows[t] : t);
}

__global__ void __launch_bounds__(kThreads) quantile_keys_kernel(ColView value, const uint32_t* __restrict__ rows, const uint32_t* __restrict__ idx,
                                                                  const uint32_t* d_m, uint64_t* __restrict__ keys) {
  const uint32_t m = *d_m;
  for (uint32_t j = blockIdx.x * kThreads + threadIdx.x; j < m; j += gridDim.x * kThreads) {
    const uint32_t t = idx[j];
    keys[j] = order_key(widen(col_raw(value, rows ? rows[t] : t), value.type), value.type);
  }
}

// first j in [0, n) with idx[j] >= t
__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t* idx, uint32_t n, uint32_t t) {
  uint32_t a = 0, b = n;
  while (a < b) { const uint32_t h = a + ((b - a) >> 1); if (idx[h] < t) a = h + 1; else b = h; }
  return a;
}

// insert rank r into the sorted distinct list s->rank[0 .. s->nr)
__device__ __forceinline__ void add_rank(QuantileLarge* s, uint32_t r) {
  uint32_t i = 0;
  while (i < s->nr && s->rank[i] < r) i++;
  if (i < s->nr && s->rank[i] == r) return;
  for (uint32_t j = s->nr; j > i; j--) s->rank[j] = s->rank[j - 1];
  s->rank[i] = r;
  s->nr++;
}

// Group g = agg rows [lo, hi): its slice [start, start + m) of the keys, and its tier, or the NULL result of a group without a value.  The
// tiers only read keys[start, start + m): groups that overlap (range windows) share one key array.
__device__ __forceinline__ void quantile_classify_group(uint32_t g, uint32_t lo, uint32_t hi, const uint32_t* __restrict__ idx, uint32_t n_vals,
                                                        const QuantileSpec& qs, uint32_t G, QuantileGroup* __restrict__ list,
                                                        QuantileLarge* __restrict__ large, uint32_t* counters, double* __restrict__ out,
                                                        uint8_t* __restrict__ valid) {
  const uint32_t start = lower_bound_u32(idx, n_vals, lo), m = lower_bound_u32(idx, n_vals, hi) - start;
  valid[g] = m > 0;
  if (m == 0) {
    for (uint32_t j = 0; j < qs.n; j++) out[size_t(j) * G + g] = 0.0;
  } else if (m <= kQuantileSmallMax) {
    list[atomicAdd(&counters[QC_SMALL], 1u)] = QuantileGroup{g, start, m};
  } else if (m <= kQuantileMediumMax) {
    list[G - 1 - atomicAdd(&counters[QC_MEDIUM], 1u)] = QuantileGroup{g, start, m};
    atomicMax(&counters[QC_MEDIUM_MAX], m);
  } else {
    // one 64-bit add takes the slot (high word) and the first chunk (low word): chunk bases grow with the slot
    const uint32_t chunks = (m + kQuantileChunk - 1) / kQuantileChunk;
    const unsigned long long at = atomicAdd(reinterpret_cast<unsigned long long*>(&counters[QC_LARGE_CHUNKS]), (1ull << 32) | chunks);
    QuantileLarge* s = &large[at >> 32];
    s->chunk = uint32_t(at);
    s->g = g;
    s->start = start;
    s->m = m;
    s->nr = 0;
    for (uint32_t j = 0; j < qs.n; j++) {
      const QRank r = quantile_rank(qs.q[j], m);
      add_rank(s, r.lo);
      add_rank(s, r.hi);
    }
    for (uint32_t i = 0; i < s->nr; i++) {
      s->left[i] = s->rank[i];
      s->prefix[i] = 0;
    }
  }
}

__global__ void quantile_classify_kernel(const uint32_t* __restrict__ seg, const uint32_t* d_g, const uint32_t* d_r,
                                                                      const uint32_t* __restrict__ idx, QuantileSpec qs, uint32_t G,
                                                                      QuantileGroup* __restrict__ list, QuantileLarge* __restrict__ large,
                                                                      uint32_t* counters, double* __restrict__ out, uint8_t* __restrict__ valid) {
  const uint32_t g_total = *d_g, r_total = *d_r, n_vals = counters[QC_VALUES];
  for (uint32_t g = blockIdx.x * kThreads + threadIdx.x; g < g_total; g += gridDim.x * kThreads) {
    const uint32_t lo = seg[g], hi = g + 1 < g_total ? seg[g + 1] : r_total;
    quantile_classify_group(g, lo, hi, idx, n_vals, qs, G, list, large, counters, out, valid);
  }
}

// The same for range windows: window w = agg rows [win_lo[w], win_hi[w]); count[w] = its rows
__global__ void quantile_classify_windows_kernel(const uint32_t* __restrict__ win_lo, const uint32_t* __restrict__ win_hi, uint32_t W,
                                                 const uint32_t* __restrict__ idx, QuantileSpec qs, QuantileGroup* __restrict__ list,
                                                 QuantileLarge* __restrict__ large, uint32_t* counters, double* __restrict__ out,
                                                 uint8_t* __restrict__ valid, uint64_t* __restrict__ count) {
  const uint32_t n_vals = counters[QC_VALUES];
  for (uint32_t w = blockIdx.x * kThreads + threadIdx.x; w < W; w += gridDim.x * kThreads) {
    const uint32_t lo = win_lo[w], hi = win_hi[w];
    count[w] = hi - lo;
    quantile_classify_group(w, lo, hi, idx, n_vals, qs, W, list, large, counters, out, valid);
  }
}

// One warp per group: lane i holds key i (the pad ~0 beyond m sorts last and is never selected: ranks stay below m), a bitonic network
// over the next power of two >= m sorts them, and lane j < Q reads the keys of its ranks lo / hi from their lanes.
__global__ void __launch_bounds__(kThreads) quantile_small_kernel(const uint64_t* __restrict__ keys, const QuantileGroup* __restrict__ list,
                                                                   const uint32_t* counters, QuantileSpec qs, uint32_t type, uint32_t G,
                                                                   double* __restrict__ out) {
  const uint32_t n = counters[QC_SMALL], lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (kThreads / 32);
  for (uint32_t i = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); i < n; i += warps) {
    const QuantileGroup gr = list[i];
    uint64_t key = lane < gr.m ? keys[gr.start + lane] : ~0ull;
    uint32_t width = 1;
    while (width < gr.m) width <<= 1;
    for (uint32_t k = 2; k <= width; k <<= 1)
      for (uint32_t j = k >> 1; j > 0; j >>= 1) {
        const uint64_t other = __shfl_xor_sync(kFull, key, j);
        const bool ascending = (lane & k) == 0, lower = (lane & j) == 0;
        key = (lower == ascending) ? (key < other ? key : other) : (key < other ? other : key);
      }
    QRank r{0, 0, 0.0};
    if (lane < qs.n) r = quantile_rank(qs.q[lane], gr.m);
    const uint64_t klo = __shfl_sync(kFull, key, r.lo), khi = __shfl_sync(kFull, key, r.hi);
    if (lane < qs.n) out[size_t(lane) * G + gr.g] = interpolate(klo, khi, r.w, type);
  }
}

// One block per group: the keys and a pad of ~0 up to the next power of two go to shared memory, a bitonic sort orders them.
__global__ void __launch_bounds__(kThreads) quantile_medium_kernel(const uint64_t* __restrict__ keys, const QuantileGroup* __restrict__ list,
                                                                    const uint32_t* counters, QuantileSpec qs, uint32_t type, uint32_t G,
                                                                    double* __restrict__ out) {
  extern __shared__ uint64_t s_keys[];
  const uint32_t n = counters[QC_MEDIUM];
  for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
    const QuantileGroup gr = list[G - 1 - i];
    uint32_t width = 2 * kQuantileSmallMax;
    while (width < gr.m) width <<= 1;
    for (uint32_t t = threadIdx.x; t < width; t += kThreads) s_keys[t] = t < gr.m ? keys[gr.start + t] : ~0ull;
    for (uint32_t k = 2; k <= width; k <<= 1)
      for (uint32_t j = k >> 1; j > 0; j >>= 1) {
        __syncthreads();
        for (uint32_t t = threadIdx.x; t < width / 2; t += kThreads) {
          const uint32_t a = ((t & ~(j - 1)) << 1) | (t & (j - 1)), b = a + j;
          const uint64_t x = s_keys[a], y = s_keys[b];
          if ((x > y) == ((a & k) == 0)) { s_keys[a] = y; s_keys[b] = x; }
        }
      }
    __syncthreads();
    if (threadIdx.x < qs.n) {
      const QRank r = quantile_rank(qs.q[threadIdx.x], gr.m);
      out[size_t(threadIdx.x) * G + gr.g] = interpolate(s_keys[r.lo], s_keys[r.hi], r.w, type);
    }
    __syncthreads();
  }
}

// The bits of the digits resolved before pass d
__device__ __forceinline__ uint64_t prefix_mask(uint32_t d) { return d == 0 ? 0ull : ~0ull << (64 - 8 * d); }

// Pass d of the large tier: one block per chunk of kQuantileChunk keys of a large group (grid-stride), so that one huge group spreads over
// the grid and many one-chunk groups do too.  Ranks with equal prefixes share the histogram of the first of them (their slot); a key
// matches at most one distinct prefix.
__global__ void __launch_bounds__(kThreads) quantile_hist_kernel(const uint64_t* __restrict__ keys, const QuantileLarge* __restrict__ large,
                                                                  const uint32_t* counters, uint32_t d, uint32_t* __restrict__ hist) {
  __shared__ uint32_t s_hist[kRanks * 256];
  __shared__ uint64_t s_prefix[kRanks];
  __shared__ uint32_t s_slot[kRanks];
  __shared__ uint32_t s_n;
  const uint32_t n_large = counters[QC_LARGE], n_chunks = counters[QC_LARGE_CHUNKS], shift = 56 - 8 * d;
  const uint64_t mask = prefix_mask(d);
  for (uint32_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    // the group of chunk c: the last one whose first chunk is <= c
    uint32_t a = 0, b = n_large;
    while (b - a > 1) { const uint32_t h = a + ((b - a) >> 1); if (large[h].chunk <= c) a = h; else b = h; }
    const QuantileLarge* s = &large[a];
    const uint32_t l = a, m = s->m, first = (c - s->chunk) * kQuantileChunk;
    __syncthreads();                                   // the previous chunk's flush is done with the shared arrays
    if (threadIdx.x == 0) {
      // the distinct prefixes, each with the slot (rank index) whose histogram it fills
      uint32_t n = 0;
      for (uint32_t r = 0; r < s->nr; r++)
        if (r == 0 || s->prefix[r] != s->prefix[r - 1]) { s_prefix[n] = s->prefix[r]; s_slot[n] = r; n++; }
      s_n = n;
    }
    __syncthreads();
    const uint32_t n = s_n;
    for (uint32_t t = threadIdx.x; t < n * 256; t += kThreads) s_hist[t] = 0;
    __syncthreads();
    const uint32_t end = m - first < kQuantileChunk ? m : first + kQuantileChunk;
    for (uint32_t t = first + threadIdx.x; t < end; t += kThreads) {
      const uint64_t key = keys[s->start + t];
      for (uint32_t p = 0; p < n; p++)
        if (((key ^ s_prefix[p]) & mask) == 0) { atomicAdd(&s_hist[p * 256 + (uint32_t(key >> shift) & 255u)], 1u); break; }
    }
    __syncthreads();
    uint32_t* h = hist + size_t(l) * kRanks * 256;
    for (uint32_t t = threadIdx.x; t < n * 256; t += kThreads)
      if (s_hist[t]) atomicAdd(&h[s_slot[t >> 8] * 256 + (t & 255u)], s_hist[t]);
  }
}

// One warp per large group resolves digit d of every rank: lane r walks its slot's histogram to the bin holding its remaining rank, then the
// warp clears the histograms for the next pass.  After the last digit the prefixes are the selected keys, and lane j < Q writes quantile j.
__global__ void __launch_bounds__(kThreads) quantile_resolve_kernel(QuantileLarge* __restrict__ large, const uint32_t* counters, uint32_t d,
                                                                     uint32_t* __restrict__ hist, QuantileSpec qs, uint32_t type, uint32_t G,
                                                                     double* __restrict__ out) {
  const uint32_t n_large = counters[QC_LARGE], lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (kThreads / 32);
  for (uint32_t l = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); l < n_large; l += warps) {
    QuantileLarge* s = &large[l];
    const uint32_t nr = s->nr;
    const uint64_t prefix = lane < nr ? s->prefix[lane] : ~0ull;
    const uint64_t prev = __shfl_up_sync(kFull, prefix, 1);
    const uint32_t starts = __ballot_sync(kFull, lane < nr && (lane == 0 || prev != prefix));
    uint32_t* h = hist + size_t(l) * kRanks * 256;
    uint64_t key = prefix;
    if (lane < nr) {
      const uint32_t slot = 31 - __clz(int(starts & (kFull >> (31 - lane))));
      const uint32_t* b = h + slot * 256;
      uint32_t left = s->left[lane], digit = 0;
      for (; digit < 255; digit++) {
        const uint32_t c = b[digit];
        if (left < c) break;
        left -= c;
      }
      key = prefix | (uint64_t(digit) << (56 - 8 * d));
      s->left[lane] = left;
      s->prefix[lane] = key;
    }
    __syncwarp();
    for (uint32_t t = lane; t < nr * 256; t += 32) h[t] = 0;
    if (d == 7) {
      // rank list positions of lane j's lo / hi
      QRank r{0, 0, 0.0};
      uint32_t ilo = 0, ihi = 0;
      if (lane < qs.n) {
        r = quantile_rank(qs.q[lane], s->m);
        while (s->rank[ilo] != r.lo) ilo++;
        while (s->rank[ihi] != r.hi) ihi++;
      }
      const uint64_t klo = __shfl_sync(kFull, key, ilo), khi = __shfl_sync(kFull, key, ihi);
      if (lane < qs.n) out[size_t(lane) * G + s->g] = interpolate(klo, khi, r.w, type);
    }
  }
}

}  // namespace

// =================================================================================================== launch wrappers
void uniform_chunk_ends(const Launch& L, const uint32_t* d_m, uint32_t batch, uint32_t nchunks, uint32_t* chunk_end) {
  if (!nchunks) return;
  uniform_chunk_ends_kernel<<<grid_for(nchunks), kThreads, 0, L.stream>>>(d_m, batch, nchunks, chunk_end);
  L.tick();
}
void clear_tail(const Launch& L, uint8_t* flags, const uint32_t* d_n, uint32_t cap) {
  if (!cap) return;
  clear_tail_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(flags, d_n, cap);
  L.tick();
}
void decode_chunks(const Launch& L, const SstDev* ssts, const RgSel* sel, uint32_t nsel, const ColSel* cols, int ncolsel,
                   uint8_t* scratch, DbaPage* dba, const uint32_t* dba_base, int* err) {
  if (!nsel || !ncolsel) return;
  decode_chunks_kernel<<<nsel * ncolsel, kThreads, 0, L.stream>>>(ssts, sel, cols, ncolsel, scratch, dba, dba_base, err);
  L.tick();
}
void dba_materialise(const Launch& L, const DbaPage* pages, uint32_t npages, const ColSel* cols, uint8_t* out) {
  if (!npages) return;
  dba_materialise_kernel<<<(npages + kDbaWarps - 1) / kDbaWarps, kDbaWarps * 32, 0, L.stream>>>(pages, npages, cols, out);
  L.tick();
}
void eval_predicates(const Launch& L, const PredSet& preds, uint32_t n, uint8_t* alive) {
  if (!n) return;
  eval_predicates_kernel<<<grid_for(n), kThreads, 0, L.stream>>>(preds, n, alive);
  L.tick();
}
void eval_binary_predicates(const Launch& L, const BinPredSet& preds, uint32_t n, bool and_alive, uint8_t* alive) {
  if (!n) return;
  eval_binary_predicates_kernel<<<grid_for(n), kThreads, preds.n_lits * sizeof(BinLitDev), L.stream>>>(preds, n, and_alive ? 1 : 0, alive);
  L.tick();
}
void eval_in_set(const Launch& L, const InSetPreds& preds, uint32_t n, bool and_alive, uint8_t* alive) {
  if (!n) return;
  eval_in_set_kernel<<<grid_for(n, int(kInSetTile)), kThreads, 0, L.stream>>>(preds, n, and_alive ? 1 : 0, alive);
  L.tick();
}
void group_map(const Launch& L, ColView col, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, const uint64_t* keys, const uint32_t* groups,
               uint32_t n_keys, uint32_t* out, int* err) {
  if (!cap) return;
  group_map_kernel<<<grid_for(cap, int(kInSetTile)), kThreads, 0, L.stream>>>(col, rows, d_r, keys, groups, n_keys, out, err);
  L.tick();
}
size_t compact_tmp_elems(uint32_t n) { return size_t(n) / kCompactTile + 2; }
void compact_flags(const Launch& L, const uint8_t* flags, uint32_t n, uint32_t* tmp, uint32_t* out_idx, uint32_t* d_total) {
  uint32_t nb = (n + kCompactTile - 1) / kCompactTile;
  if (n) { compact_count_kernel<<<grid_for(nb, 1), kThreads, 0, L.stream>>>(flags, n, tmp); L.tick(); }
  compact_scan_sums_kernel<<<1, 1024, 0, L.stream>>>(tmp, nb, d_total);
  L.tick();
  if (n) { compact_write_kernel<<<grid_for(nb, 1), kThreads, 0, L.stream>>>(flags, n, tmp, out_idx); L.tick(); }
}
void survivor_run_starts(const Launch& L, const uint32_t* surv, const uint32_t* d_m, const uint32_t* file_base, int k,
                         uint32_t* run_start) {
  survivor_run_starts_kernel<<<(k + 1 + 127) / 128, 128, 0, L.stream>>>(surv, d_m, file_base, k, run_start);
  L.tick();
}
void build_records(const Launch& L, const PkSet& pk, ColView seq, const uint32_t* surv, const uint32_t* d_m, uint32_t cap,
                   SortRec* rec) {
  if (!cap) return;
  build_records_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(pk, seq, surv, d_m, rec);
  L.tick();
}
size_t merge_split_elems(uint32_t cap) { return size_t(cap) / kMergeTile + 2; }
void merge_pass(const Launch& L, const SortRec* src, SortRec* dst, const uint32_t* run_start, int k, int level,
                const uint32_t* d_m, uint32_t cap, uint32_t* splits) {
  if (!cap) return;
  const uint32_t ntiles = (cap + kMergeTile - 1) / kMergeTile;
  merge_partition_kernel<<<grid_for(ntiles), kThreads, 0, L.stream>>>(src, run_start, k, level, d_m, splits);
  L.tick();
  merge_pass_kernel<<<grid_for(cap, kMergeTile, kNumSMs * 8), kThreads, 0, L.stream>>>(src, dst, run_start, k, level, d_m, splits);
  L.tick();
}
void records_to_rows(const Launch& L, const SortRec* rec, const uint32_t* d_m, uint32_t cap, uint32_t* order) {
  if (!cap) return;
  records_to_rows_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(rec, d_m, order);
  L.tick();
}
void dedup_flags_cols(const Launch& L, const PkSet& pk, const uint32_t* order, const uint32_t* d_m, uint32_t cap, uint8_t* keep) {
  if (!cap) return;
  dedup_flags_cols_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(pk, order, d_m, keep);
  L.tick();
}
void dedup_flags_recs(const Launch& L, const SortRec* rec, const uint32_t* d_m, uint32_t cap, uint8_t* keep) {
  if (!cap) return;
  dedup_flags_recs_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(rec, d_m, keep);
  L.tick();
}
void gather_rows(const Launch& L, const uint32_t* order, const uint32_t* out_pos, const uint32_t* d_r, uint32_t cap,
                 uint32_t* out_rows) {
  if (!cap) return;
  gather_rows_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(order, out_pos, d_r, out_rows);
  L.tick();
}
void batch_bounds(const Launch& L, const uint32_t* out_pos, const uint32_t* d_r, const uint32_t* chunk_end, uint32_t nchunks,
                  uint32_t* bound) {
  if (!nchunks) return;
  batch_bounds_kernel<<<(nchunks + 127) / 128, 128, 0, L.stream>>>(out_pos, d_r, chunk_end, nchunks, bound);
  L.tick();
}
void chunk_ends_from_rows(const Launch& L, const uint32_t* surv, const uint32_t* d_m, const uint32_t* piece_end_row,
                          uint32_t npieces, uint32_t* chunk_end) {
  if (!npieces) return;
  chunk_ends_kernel<<<(npieces + 127) / 128, 128, 0, L.stream>>>(surv, d_m, piece_end_row, npieces, chunk_end);
  L.tick();
}
void gather_column(const Launch& L, ColView src, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, void* dst_vals,
                   uint8_t* dst_valid) {
  if (!cap) return;
  int g = grid_for(cap);
  switch (src.width) {
    case 1: gather_column_kernel<uint8_t><<<g, kThreads, 0, L.stream>>>((const uint8_t*)src.vals, src.valid, rows, d_r, (uint8_t*)dst_vals, dst_valid); break;
    case 2: gather_column_kernel<uint16_t><<<g, kThreads, 0, L.stream>>>((const uint16_t*)src.vals, src.valid, rows, d_r, (uint16_t*)dst_vals, dst_valid); break;
    case 4: gather_column_kernel<uint32_t><<<g, kThreads, 0, L.stream>>>((const uint32_t*)src.vals, src.valid, rows, d_r, (uint32_t*)dst_vals, dst_valid); break;
    default: gather_column_kernel<uint64_t><<<g, kThreads, 0, L.stream>>>((const uint64_t*)src.vals, src.valid, rows, d_r, (uint64_t*)dst_vals, dst_valid);
  }
  L.tick();
}
void pack_validity(const Launch& L, const uint8_t* valid_bytes, uint32_t n, uint8_t* bitmap, unsigned long long* null_count) {
  if (!n) return;
  pack_validity_kernel<<<grid_for((n + 7) / 8), kThreads, 0, L.stream>>>(valid_bytes, n, bitmap, null_count);
  L.tick();
}
void group_flags(const Launch& L, const AggSpecDev& spec, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, uint8_t* head) {
  if (!cap) return;
  group_flags_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(spec, rows, d_r, head);
  L.tick();
}
void reduce_groups(const Launch& L, const AggSpecDev& spec, const uint32_t* rows, const uint32_t* d_r, const uint32_t* seg_start,
                   const uint32_t* d_g, uint32_t cap, AggOut out) {
  if (!cap) return;
  reduce_groups_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(spec, rows, d_r, seg_start, d_g, out);
  L.tick();
}
void reduce_counter_groups(const Launch& L, const AggSpecDev& spec, const uint32_t* rows, const uint32_t* d_r, const uint32_t* seg_start,
                           const uint32_t* d_g, uint32_t cap, CounterOut out) {
  if (!cap) return;
  reduce_counter_groups_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(spec, rows, d_r, seg_start, d_g, out);
  L.tick();
}
void pack_agg(const Launch& L, AggOut in, uint32_t gwidth, uint64_t g, uint64_t cap, long long* dst) {
  if (!cap) return;
  pack_agg_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(in, gwidth, g, cap, dst);
  L.tick();
}
void gather_lens(const Launch& L, ColView col, const uint32_t* rows, const uint32_t* d_n, uint32_t cap, uint32_t* out) {
  if (!cap) return;
  gather_lens_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(col, rows, d_n, cap, out);
  L.tick();
}
void copy_var(const Launch& L, ColView col, const uint32_t* rows, const uint32_t* d_n, uint32_t cap, const uint32_t* offs, uint8_t* dst) {
  if (!cap) return;
  copy_var_kernel<<<grid_for(uint64_t(cap) * 32), kThreads, 0, L.stream>>>(col, rows, d_n, offs, dst);
  L.tick();
}
void first_rows(const Launch& L, const uint32_t* order, const uint32_t* out_pos, const uint32_t* d_r, uint32_t cap, uint32_t* out) {
  if (!cap) return;
  first_rows_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(order, out_pos, d_r, out);
  L.tick();
}
void run_offsets(const Launch& L, const uint32_t* cum, const uint32_t* out_pos, const uint32_t* d_r, const uint32_t* d_m, uint32_t cap, uint32_t* out) {
  run_offsets_kernel<<<grid_for(uint64_t(cap) + 1), kThreads, 0, L.stream>>>(cum, out_pos, d_r, d_m, out);
  L.tick();
}
void append_validity(const Launch& L, ColView col, const uint32_t* order, const uint32_t* out_pos, const uint32_t* d_r, const uint32_t* run_offs,
                     uint32_t cap, uint8_t* valid, int* err) {
  if (!cap) return;
  append_validity_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(col, order, out_pos, d_r, run_offs, valid, err);
  L.tick();
}
void exclusive_scan_u32(const Launch& L, uint32_t* data, uint32_t n, uint32_t* d_total) {
  compact_scan_sums_kernel<<<1, 1024, 0, L.stream>>>(data, n, d_total);
  L.tick();
}
void fill_u32(const Launch& L, uint32_t* p, uint32_t v, uint32_t n) {
  if (!n) return;
  fill_u32_kernel<<<grid_for(n), kThreads, 0, L.stream>>>(p, v, n);
  L.tick();
}

// quantiles per group
size_t quantile_large_cap(uint32_t cap) { return size_t(cap) / (kQuantileMediumMax + 1) + 1; }
size_t quantile_hist_elems(uint32_t n_large) { return size_t(n_large) * kRanks * 256; }

// the non-NULL agg rows (b.idx) and their order keys (b.keys), in agg-row order
static void quantile_value_keys(const Launch& L, ColView value, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, const QuantileBufs& b) {
  quantile_flags_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(value, rows, d_r, cap, b.flags);
  L.tick();
  compact_flags(L, b.flags, cap, b.compact_tmp, b.idx, b.counters + QC_VALUES);
  quantile_keys_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(value, rows, b.idx, b.counters + QC_VALUES, b.keys);
  L.tick();
}

void quantile_prepare(const Launch& L, ColView value, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, const uint32_t* seg,
                      const uint32_t* d_g, uint32_t G, const QuantileSpec& qs, const QuantileBufs& b) {
  if (!cap || !G) return;
  quantile_value_keys(L, value, rows, d_r, cap, b);
  quantile_classify_kernel<<<grid_for(G), kThreads, 0, L.stream>>>(seg, d_g, d_r, b.idx, qs, G, b.list, b.large, b.counters, b.out, b.valid);
  L.tick();
}

void quantile_prepare_windows(const Launch& L, ColView value, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, const uint32_t* win_lo,
                              const uint32_t* win_hi, uint32_t W, const QuantileSpec& qs, const QuantileBufs& b, uint64_t* count) {
  if (!cap || !W) return;
  quantile_value_keys(L, value, rows, d_r, cap, b);
  quantile_classify_windows_kernel<<<grid_for(W), kThreads, 0, L.stream>>>(win_lo, win_hi, W, b.idx, qs, b.list, b.large, b.counters, b.out,
                                                                           b.valid, count);
  L.tick();
}

// range windows
size_t range_block_elems(uint32_t cap) { return size_t(cap) / kRangeTile + 2; }

void range_count(const Launch& L, const RangeSpecDev& rs, ColView ts, ColView value, const uint32_t* rows, const uint32_t* d_r, uint32_t cap,
                 const uint8_t* head, const RangeBufs& b) {
  if (!cap) return;
  range_gather_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(ts, value, rows, d_r, b.ts, b.v, b.ok);
  L.tick();
  const int blocks = grid_for((cap + kRangeTile - 1) / kRangeTile, 1);
  range_count_kernel<<<blocks, kThreads, 0, L.stream>>>(rs, b.ts, head, d_r, b.off, b.wsum, b.msum);
  L.tick();
  range_scan_sums_kernel<<<1, kThreads, 0, L.stream>>>(b.wsum, b.msum, d_r, b.totals);
  L.tick();
}

void range_windows(const Launch& L, const RangeSpecDev& rs, const uint32_t* d_r, uint32_t cap, const uint8_t* head, const uint32_t* seg, uint32_t G,
                   ColView group, const uint32_t* rows, uint32_t W, const RangeBufs& b, RangeWindows out) {
  if (!cap || !W) return;
  range_offsets_kernel<<<grid_for((cap + kRangeTile - 1) / kRangeTile, 1), kThreads, 0, L.stream>>>(b.wsum, d_r, b.off);
  L.tick();
  range_windows_kernel<<<grid_for(W), kThreads, 0, L.stream>>>(rs, b.ts, head, b.off, d_r, seg, G, group, rows, W, out);
  L.tick();
}

void reduce_range_windows(const Launch& L, const RangeBufs& b, const uint32_t* win_lo, const uint32_t* win_hi, uint32_t W, RangeOut out) {
  if (!W) return;
  reduce_range_windows_kernel<<<grid_for(W), kThreads, 0, L.stream>>>(b.ts, b.v, b.ok, win_lo, win_hi, W, out);
  L.tick();
}

void range_function(const Launch& L, const RangeFnSpec& f, const RangeBufs& b, const uint32_t* win_lo, const uint32_t* win_hi, const int64_t* win_t,
                    uint32_t W, double* value, uint8_t* valid) {
  if (!W) return;
  range_function_kernel<<<grid_for(W), kThreads, 0, L.stream>>>(f, b.ts, b.v, b.ok, win_lo, win_hi, win_t, W, value, valid);
  L.tick();
}

void range_fn_gather(const Launch& L, const uint32_t* idx, const uint32_t* d_n, uint32_t cap, ColView key, const int64_t* t, const double* value,
                     void* key_out, int64_t* t_out, double* value_out) {
  if (!cap) return;
  range_fn_gather_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(idx, d_n, key, t, value, key_out, t_out, value_out);
  L.tick();
}

void range_fn_sort_keys(const Launch& L, const uint32_t* idx, const uint32_t* d_n, uint32_t cap, const uint32_t* ordinal, const int64_t* t,
                        int64_t start, int64_t step, int shift, uint64_t* keys, uint32_t* vals) {
  if (!cap) return;
  range_fn_sort_keys_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(idx, d_n, ordinal, t, start, step, shift, keys, vals);
  L.tick();
}

void topk_rank_keys(const Launch& L, const uint32_t* idx, const uint32_t* d_n, uint32_t cap, const double* value, bool descending, uint64_t* keys) {
  if (!cap) return;
  topk_rank_keys_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(idx, d_n, value, descending ? 1 : 0, keys);
  L.tick();
}

void topk_keep(const Launch& L, const uint32_t* seg, const uint32_t* d_n, uint32_t cap, uint32_t k, uint8_t* keep) {
  if (!cap) return;
  topk_keep_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(seg, d_n, cap, k, keep);
  L.tick();
}

void topk_gather(const Launch& L, const uint32_t* pos, const uint32_t* d_r, uint32_t cap, const uint32_t* win, const uint32_t* ordinal, const int64_t* t,
                 const double* value, const uint32_t* win_lo, ColView series, const uint32_t* rows, TopkOut out) {
  if (!cap) return;
  topk_gather_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(pos, d_r, win, ordinal, t, value, win_lo, series, rows, out);
  L.tick();
}

void histogram_sort_keys(const Launch& L, const uint32_t* idx, const uint32_t* d_n, uint32_t cap, const uint32_t* ordinal, const BucketPair* pair,
                         const int64_t* t, int64_t start, int64_t step, int shift, int lbits, uint64_t* keys, uint32_t* vals) {
  if (!cap) return;
  histogram_sort_keys_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(idx, d_n, ordinal, pair, t, start, step, shift, lbits, keys, vals);
  L.tick();
}

void histogram_heads(const Launch& L, const uint32_t* ordinal, const int64_t* t, const BucketPair* pair, const uint32_t* d_n, uint32_t cap,
                     uint8_t* head) {
  if (!cap) return;
  histogram_heads_kernel<<<grid_for(cap), kThreads, 0, L.stream>>>(ordinal, t, pair, d_n, head);
  L.tick();
}

void histogram_quantile(const Launch& L, const QuantileSpec& qs, const uint32_t* seg, uint32_t S, uint32_t n, const uint32_t* ordinal,
                        const int64_t* t, double* count, const BucketPair* pair, const double* bounds, const uint32_t* group_ordinal, HistogramOut out) {
  if (!S) return;
  histogram_quantile_kernel<<<grid_for(S), kThreads, 0, L.stream>>>(qs, seg, S, n, ordinal, t, count, pair, bounds, group_ordinal, out);
  L.tick();
}

void quantile_select(const Launch& L, const QuantileSpec& qs, uint32_t type, uint32_t G, const uint32_t host_counters[kQuantileCounters],
                     const QuantileBufs& b) {
  const uint32_t n_small = host_counters[QC_SMALL], n_medium = host_counters[QC_MEDIUM], n_large = host_counters[QC_LARGE];
  if (n_small) {
    quantile_small_kernel<<<grid_for(n_small, kThreads / 32), kThreads, 0, L.stream>>>(b.keys, b.list, b.counters, qs, type, G, b.out);
    L.tick();
  }
  if (n_medium) {
    uint32_t width = 2 * kQuantileSmallMax;
    while (width < host_counters[QC_MEDIUM_MAX]) width <<= 1;
    quantile_medium_kernel<<<grid_for(n_medium, 1), kThreads, width * sizeof(uint64_t), L.stream>>>(b.keys, b.list, b.counters, qs, type, G,
                                                                                                       b.out);
    L.tick();
  }
  if (n_large) {
    const int hist_blocks = grid_for(host_counters[QC_LARGE_CHUNKS], 1);
    for (uint32_t d = 0; d < 8; d++) {
      quantile_hist_kernel<<<hist_blocks, kThreads, 0, L.stream>>>(b.keys, b.large, b.counters, d, b.hist);
      L.tick();
      quantile_resolve_kernel<<<grid_for(n_large, kThreads / 32), kThreads, 0, L.stream>>>(b.large, b.counters, d, b.hist, qs, type, G, b.out);
      L.tick();
    }
  }
}

}  // namespace k
}  // namespace horae
