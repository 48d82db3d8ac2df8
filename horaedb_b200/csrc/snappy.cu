// snappy.cu — raw-Snappy page decompression kernels.  The decoder itself (one warp per page: binary-lifting parse of a staged
// window, word mode / run mode execution, ring -> global flushes) lives in snappy_core.h, which the CPU test-suite compiles too.
#include "kernels.h"
#include "chunk_scratch.h"

#include <cstdlib>
#include <cstring>

#define SNP_FN __device__ __forceinline__
#define snp_shfl(v, src) __shfl_sync(0xffffffffu, (v), (src))
#define snp_shfl_up(v, d) __shfl_up_sync(0xffffffffu, (v), (d))
#define snp_ballot(p) __ballot_sync(0xffffffffu, (p))
#define snp_any(p) __any_sync(0xffffffffu, (p))
#define snp_syncwarp() __syncwarp()
#define snp_ldg8(p) __ldg(p)
#define snp_ldg64(p) __ldg(p)
#define snp_funnel_r(lo, hi, sh) __funnelshift_r((lo), (hi), (sh))
#define snp_byte_perm(a, b, s) __byte_perm((a), (b), (s))
#define snp_ffs(x) __ffs(x)
#define SNP_HAVE_LDCG64 1
#define snp_set_err(err, code) atomicExch((err), (code))
namespace horae {
namespace snp {
__device__ __forceinline__ uint32_t snp_ldcg32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ uint64_t snp_ldcg64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ uint8_t snp_ldcg8(const uint8_t* p) {
  uint32_t v;
  asm volatile("ld.global.cg.u8 %0, [%1];" : "=r"(v) : "l"(p));
  return uint8_t(v);
}
}  // namespace snp
}  // namespace horae
#include "snappy_core.h"

namespace horae {
namespace k {

namespace {

using namespace horae::snp;
constexpr int kWarpsPerCta = 4;

__device__ __forceinline__ void init_tag_tables(uint8_t* s_csz, uint32_t* s_lut) {
  for (uint32_t t = threadIdx.x; t < 256; t += kWarpsPerCta * 32) { s_csz[t] = uint8_t(elem_csize(t)); s_lut[t] = elem_lut(t); }
  __syncthreads();
}

// The pages of one column chunk (entry ci of the job) into its scratch: a compressed dictionary page first (p == -1), then the data
// pages.  ONE call site of the decoder per kernel keeps the kernel's code (and its instruction-cache footprint) at one copy.
__device__ __forceinline__ void decode_chunk(const SnappyJob& J, const RgSel& rs, const SstDev& sst, const ChunkDev* chunks, const ChunkDev& ch,
                                             int ci, WarpSmem& sm, uint32_t& phase, const uint8_t* s_csz, const uint32_t* s_lut, int lane) {
  uint8_t* dst = J.scratch + (J.fixed_stride ? rs.scratch_off + uint64_t(J.region[ci]) * J.fixed_stride
                                             : chunk_scratch_off(rs, chunks, J.cols, ci));
  const bool vmode = ch.phys == PT_INT64 || ch.phys == PT_DOUBLE;         // 8-byte values: value mode
  for (int p = ch.dict_uncomp ? -1 : 0; p < int(ch.num_pages); p++) {
    const uint8_t* src;
    uint32_t n, ulen, stop_at = 0xffffffffu;
    uint64_t advance;
    bool compressed = true;
    if (p < 0) {
      src = sst.bytes + ch.dict_payload_off; n = ch.dict_comp; ulen = ch.dict_uncomp;
      advance = dict_scratch(ch.codec, ch.phys, ch.dict_uncomp);
    } else {
      const PageDev pg = sst.pages[ch.first_page + p];
      const PageStream ps = page_stream(pg);
      src = sst.bytes + pg.payload_off + ps.skip; n = ps.comp; ulen = ps.out;
      compressed = ps.compressed;
      if (J.partial[ci]) {
        // the consumer reads rows [0, rs.out_row) only (gate-first: nothing behind the last row that passes the gate column can
        // survive the filter).  The page is all-valid PLAIN: its values end at the page end, behind a level prefix of any length (one RLE
        // run, or many runs: other writers' all-valid levels can take more bytes than rows), so the needed ones end num_rows - out_row
        // values before it.  The stop is the later of that and the front estimate (a prefix of <= 16 + rows / 8 bytes), so a page whose
        // values do not end at its end still decodes at least as far as before
        const uint32_t w = (ch.phys == 1 || ch.phys == 4) ? 4u : 8u;
        const uint64_t tail = uint64_t(rs.num_rows - rs.out_row) * w;
        const uint32_t front = 16u + (rs.num_rows + 7u) / 8u + 8u + rs.out_row * w;
        const uint32_t back = tail < ulen ? uint32_t(ulen - tail) : ulen;
        stop_at = front > back ? front : back;
      }
      advance = page_body_scratch(ch.codec, pg) + page_image_scratch(pg);
    }
    if (compressed) snappy_page(src, n, dst, ulen, stop_at, sm, phase, s_csz, s_lut, lane, J.err, vmode);
    dst += advance;
  }
}

// One warp per column chunk, chunks handed out by an atomic ticket in the order (column order[0] of every row group,
// then order[1], ...): the host lists the columns with the most compressed bytes first, and inside a column J.lpt lists
// the row groups with the most bytes to decode first, so the long pages start early and the short ones fill the tail.
__global__ void __launch_bounds__(kWarpsPerCta * 32, 7) snappy_pages_kernel(const __grid_constant__ SnappyJob J) {
  __shared__ WarpSmem s_w[kWarpsPerCta];
  __shared__ uint32_t s_lut[256];
  __shared__ uint8_t s_csz[256];
  init_tag_tables(s_csz, s_lut);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  WarpSmem& sm = s_w[wid];
  bulk_init(sm, lane);
  uint32_t phase = 0;
  const uint32_t nsel = J.d_nsel ? *J.d_nsel : J.nsel;
  const uint32_t nchunks = nsel * uint32_t(J.ncols);
  for (;;) {
    uint32_t c = 0;
    if (lane == 0) c = atomicAdd(J.ticket, 1u);
    c = __shfl_sync(0xffffffffu, c, 0);
    if (c >= nchunks) return;
    const uint32_t si = J.lpt ? J.lpt[c % nsel] : c % nsel;
    const int ci = J.order[c / nsel];
    RgSel rs = J.sel[si];
    SstDev sst = J.ssts[rs.sst];
    const ChunkDev* chunks = sst.chunks + size_t(rs.rg) * sst.ncols;
    ChunkDev ch = chunks[J.col_from_cols ? J.cols[ci].col : J.col[ci]];
    if (ch.codec != CODEC_SNAPPY) continue;
    if (ch.stored && J.skip_stored[ci]) continue;                 // read in place by the consumer
    decode_chunk(J, rs, sst, chunks, ch, ci, sm, phase, s_csz, s_lut, lane);
  }
}

// pages given by pointer (transient loads decompress the gate column before the SST's tables exist on the device)
__global__ void __launch_bounds__(kWarpsPerCta * 32, 8) snappy_raw_kernel(const RawPage* __restrict__ pages, uint32_t n, unsigned int* ticket, int* err) {
  __shared__ WarpSmem s_w[kWarpsPerCta];
  __shared__ uint32_t s_lut[256];
  __shared__ uint8_t s_csz[256];
  init_tag_tables(s_csz, s_lut);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  bulk_init(s_w[wid], lane);
  uint32_t phase = 0;
  for (;;) {
    uint32_t c = 0;
    if (lane == 0) c = atomicAdd(ticket, 1u);
    c = __shfl_sync(0xffffffffu, c, 0);
    if (c >= n) return;
    const RawPage pg = pages[c];
    // a RawPage does not say its value width: word and run mode only
    snappy_page(pg.src, pg.comp_size, pg.dst, pg.uncomp_size, 0xffffffffu, s_w[wid], phase, s_csz, s_lut, lane, err, false);
  }
}

// Gate-first fused scans over a 4-byte gate column: the row-group gate straight from the gate column's compressed pages, one warp per
// selected row group.  Writes what the scan needs of the column and nothing else: one bit per row (bit r & 31 of word r >> 5 at
// scratch + scratch_off + bits_off, bits past the last row zero), flags[si] = the row group has a passing row, and sel[si].out_row = the
// last passing row + 2 (capped at the row count; 0 without one).  A single compressed page is taken in the bit domain
// (snappy_gate_page); any other chunk — or a page that path declines — is decompressed into the column's scratch region as
// snappy_pages_kernel does and its values are tested there, with the same result.
__global__ void __launch_bounds__(kWarpsPerCta * 32, 7) snappy_gate_kernel(const __grid_constant__ GateJob G) {
  __shared__ WarpSmem s_w[kWarpsPerCta];
  __shared__ uint32_t s_lut[256];
  __shared__ uint8_t s_csz[256];
  init_tag_tables(s_csz, s_lut);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  WarpSmem& sm = s_w[wid];
  bulk_init(sm, lane);
  uint32_t phase = 0;
  const SnappyJob& J = G.J;
  const uint32_t nsel = *J.d_nsel;
  const GateTest g{G.flip, G.lo, G.span};
  for (;;) {
    uint32_t si = 0;
    if (lane == 0) si = atomicAdd(J.ticket, 1u);
    si = __shfl_sync(0xffffffffu, si, 0);
    if (si >= nsel) return;
    const RgSel rs = J.sel[si];
    const SstDev sst = J.ssts[rs.sst];
    const ChunkDev* chunks = sst.chunks + size_t(rs.rg) * sst.ncols;
    const ChunkDev ch = chunks[J.col[0]];
    const uint32_t nrows = rs.num_rows, nw = (nrows + 31) >> 5;
    uint32_t* bits = reinterpret_cast<uint32_t*>(J.scratch + rs.scratch_off + G.bits_off);
    const PageDev pg = sst.pages[ch.first_page];
    uint32_t last = 0;
    bool done = false;
    if (ch.codec == CODEC_SNAPPY && ch.num_pages == 1 && !ch.dict_uncomp) {
      const PageStream ps = page_stream(pg);
      if (ps.compressed)
        done = snappy_gate_page(sst.bytes + pg.payload_off + ps.skip, ps.comp, ps.out, ch.optional != 0, nrows, g, sm, phase, s_csz, s_lut,
                                lane, &last);
      if (done) {
        const GateTab& t = gate_tab(sm);
        for (uint32_t w = lane; w < nw; w += 32) bits[w] = t.bits[w];
      }
    }
    if (!done) {
      if (ch.codec == CODEC_SNAPPY) {
        if (lane == 0) atomicAdd(G.fallback, 1u);
        decode_chunk(J, rs, sst, chunks, ch, 0, sm, phase, s_csz, s_lut, lane);
        __syncwarp();
      }
      // the values where the fused scan would find them (slot_base_chase): the scratch region, or the file's page; behind the level prefix
      const uint8_t* base = ch.codec == CODEC_SNAPPY ? J.scratch + rs.scratch_off + uint64_t(J.region[0]) * J.fixed_stride
                                                     : sst.bytes + pg.payload_off;
      if (ch.optional) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(base);
        const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
        uint32_t lv = snp_funnel_r(snp_ldcg32(q), snp_ldcg32(q + 1), uint32_t(a & 3) * 8);
        if (lv > pg.uncomp_size) { lv = 0; if (lane == 0) atomicExch(J.err, 202); }
        base += 4 + lv;
      }
      const uintptr_t a = reinterpret_cast<uintptr_t>(base);
      const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
      const uint32_t sh = uint32_t(a & 3) * 8;
      for (uint32_t w = 0; w < nw; w++) {
        const uint32_t i = w * 32 + lane;
        const bool pass = i < nrows && gate_pass(g, sh ? snp_funnel_r(snp_ldcg32(q + i), snp_ldcg32(q + i + 1), sh) : snp_ldcg32(q + i));
        if (pass) last = i + 1;
        const uint32_t b = __ballot_sync(0xffffffffu, pass);
        if (lane == 0) bits[w] = b;
      }
      for (int d = 16; d > 0; d >>= 1) { const uint32_t o = __shfl_xor_sync(0xffffffffu, last, d); last = o > last ? o : last; }
    }
    if (lane == 0) {
      G.flags[si] = last ? 1 : 0;
      G.sel[si].out_row = last ? (last + 1 < nrows ? last + 1 : nrows) : 0;
    }
  }
}

}  // namespace

// Resident CTAs per SM the decompression kernels ask for.  8 would fill an SM's 228 KB of shared memory (8 x (27.3 + 1) KB); 7 gave the
// fastest decompression stage on one H100 SXM at a 400 W power limit (bench config 2, alternating runs: 6 -> 1.83, 7 -> 1.73, 8 -> 1.76 ms
// per step: the stage is bound by instruction issue and shared-memory traffic, not by the number of warps), and ~30 KB per SM stay free
// for the library's own NCCL all-gather of the previous step's partials, which runs NEXT to the decompression of the current step
// (hg_agg_combine).  snappy_pages_kernel is compiled for 7 (72 registers: value mode's state fits without spilling).
// HORAE_SNAPPY_CTAS_PER_SM overrides it for A/B timing.
static uint32_t snappy_max_ctas() {
  static const int env = getenv("HORAE_SNAPPY_CTAS_PER_SM") ? atoi(getenv("HORAE_SNAPPY_CTAS_PER_SM")) : 0;
  int n = env > 0 ? env : 7;
  if (n > 8) n = 8;
  return uint32_t(kNumSMs) * uint32_t(n);
}

void snappy_raw_pages(const Launch& L, const RawPage* d_pages, uint32_t n, unsigned int* ticket, int* err) {
  if (!n) return;
  uint32_t ctas = (n + kWarpsPerCta - 1) / kWarpsPerCta;
  if (ctas > snappy_max_ctas()) ctas = snappy_max_ctas();
  snappy_raw_kernel<<<ctas, kWarpsPerCta * 32, 0, L.stream>>>(d_pages, n, ticket, err);
  L.tick();
}

void snappy_pages(const Launch& L, const SnappyJob& job, uint32_t max_chunks) {
  if (!max_chunks) return;
  uint32_t ctas = (max_chunks + kWarpsPerCta - 1) / kWarpsPerCta;
  if (ctas > snappy_max_ctas()) ctas = snappy_max_ctas();
  snappy_pages_kernel<<<ctas, kWarpsPerCta * 32, 0, L.stream>>>(job);
  L.tick();
}

void snappy_gate_pages(const Launch& L, const GateJob& job, uint32_t max_rgs) {
  if (!max_rgs) return;
  uint32_t ctas = (max_rgs + kWarpsPerCta - 1) / kWarpsPerCta;
  if (ctas > snappy_max_ctas()) ctas = snappy_max_ctas();
  snappy_gate_kernel<<<ctas, kWarpsPerCta * 32, 0, L.stream>>>(job);
  L.tick();
}

void snappy_chunks(const Launch& L, const SstDev* ssts, const RgSel* sel, uint32_t nsel, const ColSel* cols, int ncolsel,
                   uint8_t* scratch, unsigned int* ticket, int* err) {
  if (!nsel || !ncolsel) return;
  SnappyJob J;
  std::memset(&J, 0, sizeof(J));
  J.ssts = ssts; J.sel = sel; J.d_nsel = nullptr; J.nsel = nsel; J.cols = cols; J.ncols = ncolsel;
  J.scratch = scratch; J.ticket = ticket; J.err = err; J.fixed_stride = 0;
  for (int i = 0; i < ncolsel && i < kSnappyMaxCols; i++) J.order[i] = uint8_t(i);
  J.col_from_cols = 1;      // general pipeline: column ids and the variable scratch layout come from the ColSel table
  snappy_pages(L, J, nsel * uint32_t(ncolsel));
}

}  // namespace k
}  // namespace horae
