// zstd.cu — Zstandard page decompression (ParquetCompression::Zstd, config.rs:78-94) for the general pipeline.  The decoder is
// zstd_core.h (one source for the GPU and for the CPU warp emulator of the tests); this file is the kernel around it: one warp per
// column chunk, chunks handed out by an atomic ticket, pages decompressed into the chunk's scratch where decode_chunks_kernel reads
// them (chunk_scratch.h); the chunk's literal buffer sits at the end of its scratch.
#include "kernels.h"
#include "chunk_scratch.h"

#include <cstring>

#define SNP_FN __device__ __forceinline__
#define SNP_CONST __constant__ const
#define snp_any(p) __any_sync(0xffffffffu, (p))
#define snp_syncwarp() __syncwarp()
#define snp_ldg8(p) __ldg(p)
#define snp_set_err(err, code) atomicExch((err), (code))
namespace horae {
namespace zst {
__device__ __forceinline__ uint8_t snp_ldcg8(const uint8_t* p) {
  uint32_t v;
  asm volatile("ld.global.cg.u8 %0, [%1];" : "=r"(v) : "l"(p));
  return uint8_t(v);
}
// 8 read-only input bytes at any alignment (two aligned words + funnel)
__device__ __forceinline__ uint64_t snp_ldg64u(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint64_t* q = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
  const uint32_t sh = uint32_t(a & 7) * 8;
  const uint64_t lo = __ldg(q), hi = __ldg(q + 1);
  return (lo >> sh) | ((hi << 1) << (63 - sh));
}
}  // namespace zst
}  // namespace horae
#include "zstd_core.h"

namespace horae {
namespace k {

namespace {

constexpr int kWarpsPerCta = 3;        // 14.8 KB of tables + output ring per warp: 3 warps keep the CTA under the 48 KB static limit, 5 CTAs per SM

static_assert(kZstdLitMax == zst::kBlockMax, "the literal buffer holds one block's literals");

__global__ void __launch_bounds__(kWarpsPerCta * 32) zstd_chunks_kernel(const SstDev* __restrict__ ssts, const RgSel* __restrict__ sel, uint32_t nsel,
                                                                       const ColSel* __restrict__ cols, int ncols, uint8_t* __restrict__ scratch,
                                                                       unsigned int* ticket, int* err) {
  __shared__ zst::WarpSmem s_w[kWarpsPerCta];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  zst::WarpSmem& sm = s_w[wid];
  const uint32_t nchunks = nsel * uint32_t(ncols);
  for (;;) {
    uint32_t c = 0;
    if (lane == 0) c = atomicAdd(ticket, 1u);
    c = __shfl_sync(0xffffffffu, c, 0);
    if (c >= nchunks) return;
    const uint32_t si = c % nsel;
    const int ci = int(c / nsel);
    const RgSel rs = sel[si];
    const SstDev sst = ssts[rs.sst];
    const ChunkDev* chunks = sst.chunks + size_t(rs.rg) * sst.ncols;
    const ChunkDev ch = chunks[cols[ci].col];
    if (ch.codec != CODEC_ZSTD) continue;
    uint8_t* const base = scratch + chunk_scratch_off(rs, chunks, cols, ci);
    uint8_t* dst = base;
    uint8_t* const lit = base + ch.scratch_bytes - zstd_lit_scratch(ch.dict_uncomp, sst.pages + ch.first_page, ch.num_pages);   // at the end
    for (int p = ch.dict_uncomp ? -1 : 0; p < int(ch.num_pages); p++) {
      const uint8_t* src;
      uint32_t n, ulen;
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
        advance = page_body_scratch(ch.codec, pg) + page_image_scratch(pg);
      }
      if (compressed) zst::zstd_page(src, n, dst, ulen, lit, sm, lane, err);
      __syncwarp();
      dst += advance;
    }
  }
}

}  // namespace

void zstd_chunks(const Launch& L, const SstDev* ssts, const RgSel* sel, uint32_t nsel, const ColSel* cols, int ncolsel, uint8_t* scratch,
                 unsigned int* ticket, int* err) {
  if (!nsel || !ncolsel) return;
  const uint32_t chunks = nsel * uint32_t(ncolsel);
  uint32_t ctas = (chunks + kWarpsPerCta - 1) / kWarpsPerCta;
  if (ctas > kNumSMs * 5u) ctas = kNumSMs * 5u;
  zstd_chunks_kernel<<<ctas, kWarpsPerCta * 32, 0, L.stream>>>(ssts, sel, nsel, cols, ncolsel, scratch, ticket, err);
  L.tick();
}

}  // namespace k
}  // namespace horae
