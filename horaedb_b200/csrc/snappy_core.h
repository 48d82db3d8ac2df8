// snappy_core.h — the warp-level raw-Snappy page decoder (Parquet SNAPPY codec: parquet 53.2 -> snap 1.1.1 in the reference,
// Cargo.lock:3145; format restated from the published Snappy format description).
//
// This header is the decoder's single source: snappy.cu compiles it for sm_90a (the product), and the CPU test-suite compiles
// the SAME text with the warp primitives below mapped onto 32 coroutines (tests/emu/snappy_emu.cpp; snappy_value_emu.cpp with value mode), so the lane-level logic is
// checked without a GPU.  The includer provides, before including:
//   SNP_FN                          function qualifiers (__device__ __forceinline__ / inline)
//   snp_shfl(v, src)  snp_shfl_up(v, d)  snp_ballot(pred)  snp_any(pred)  snp_syncwarp()      full-warp collectives (32-bit values)
//   snp_ldg8(p)  snp_ldg64(p)       read-only input loads (uint8_t / aligned uint64_t)
//   snp_ldcg8(p) snp_ldcg32(p)      coherent loads of this page's earlier OUTPUT (written by other lanes of the warp); an includer
//                                   that defines SNP_HAVE_LDCG64 also provides snp_ldcg64(p) (one aligned 64-bit load)
//   snp_funnel_r(lo, hi, sh)        32-bit funnel shift right (sh < 32),  snp_byte_perm(a, b, sel),  snp_ffs(x)
//   snp_set_err(err, code)
//
// Snappy is byte-serial by definition: an element's position depends on all element lengths before it, and a copy may
// read bytes produced by the element just before it.  One warp owns one page and breaks both dependencies:
//
//   parse    a 256-byte window of the compressed stream is staged in shared memory; every byte position computes
//            "where would the next element start if one started here" (J1, from a tag-byte table), four doubling steps give
//            J2..J16, and lane k finds the start of the k-th element after ANY start position with 5 dependent lookups
//            (binary lifting): 32 elements are decoded per step instead of one, and a batch may end after any element.
//            Lane l owns the 8 positions [8l, 8l+8): a table row is one 64-bit store per lane and level, built in registers.
//   execute  the longest prefix of the batch that one of two modes can take:
//     word mode   elements of <= 8 bytes (fixed-width numeric columns compress to literal(1-2) + copy(6-7) pairs): every
//                 lane builds its element's bytes in ONE 64-bit register — from the staged literal, from the ring / the
//                 page's earlier output, or from an earlier element of the same batch (parent links collapsed with five
//                 register shuffles) — and drops them into a shared-memory ring.  An element whose source straddles
//                 two elements of the batch simply ends the prefix: it starts the next batch, where its source is old.
//   staging  the compressed bytes travel global -> shared by cp.async.bulk + mbarrier, one region ahead of the parser.
//     run mode    a long element, or a run of copies with one offset (RLE-like columns: 64-byte copies at offset 4/8):
//                 out[x] = out[x - off] over the union, i.e. one periodic pattern; for off in {1,2,4,8} that is a single
//                 64-bit word stored to every aligned word of the run.
//     value mode  (pages of 8-byte values, tried first) a value run compresses to one (literal of L <= 4 bytes, copy of 8 - L
//                 bytes at an offset that is a multiple of 8) pair per value.  Lane k takes the k-th pair (element 2k, via J2..J32):
//                 its value lands at o + 8k with no prefix sum, a copy whose source value is in the batch names its parent lane
//                 exactly, an older source is ONE value-aligned 8-byte read, chains are collapsed by pointer jumping on one 32-bit
//                 word per lane (parent | L | literal bytes 1..3; byte 0 is always the lane's own), and every lane stores one aligned
//                 64-bit ring word: 32 values = 256 output bytes per step.  The ballot of the per-lane checks is the prefix it takes;
//                 anything else (level prefix, a copy spanning two values, long literals) is left to the other modes, and a word-mode
//                 step that follows ends right before the last pair it sees, so value mode picks up again on the next step.
//   flush    the ring is written to global memory in whole 32-byte sectors, 256 bytes per warp instruction.
//   literals longer than 60 bytes (incompressible columns are one literal per 64 KiB block) are plain warp copies.
#pragma once
#include <cstdint>

#ifndef SNP_STAT
#define SNP_STAT(counter, amount)      // the emulator counts windows / steps / elements here
#endif
#ifndef SNP_STAT_VALUE
#define SNP_STAT_VALUE(amount)         // value-mode steps (counted by the value-mode emulator)
#endif

namespace horae {
namespace snp {

constexpr int kWin = 256;          // compressed-stream window covered by the jump tables (bytes)
constexpr int kWinPad = 16;        // staged beyond the window: header + payload of a <= 8-byte element that starts near its end
constexpr int kRing = 4096;        // ring buffer of the most recent output (power of two)
constexpr int kHist = 2048;        // bytes before the current batch that are guaranteed to still be in the ring
constexpr int kLevels = 6;         // J1, J2, J4, J8, J16 (the next batch starts right after the last executed element), J32 (value mode)
constexpr int kMinValues = 8;      // value mode takes a batch only when at least this many value pairs line up (else word mode)
constexpr uint32_t kExit = 0xff;   // "leaves the window"; window positions are one byte per table entry
constexpr uint32_t kRestage = kWin - 80;   // start a new window when a batch would begin beyond this position (176: 14 % fewer windows than 160 on ts pages, same number of steps)
constexpr uint32_t kFlushAt = 512;         // ring -> global once this many bytes are pending (two 8-byte words per lane)
constexpr uint64_t kFill = 0xfcfcfcfcfcfcfcfcull;   // tag of a long literal: what positions behind the stream's end are staged as

// 256-byte aligned, every jump table on a 256-byte boundary: a table address is the block's base with the index as its low
// byte, i.e. ONE byte-permute (index extraction and address formation together) in front of the load.
constexpr int kStage = 448;        // bytes per staging buffer of the compressed stream (multiple of 16: bulk-copy granularity)
constexpr uint32_t kAhead = kRestage;      // the next window starts more than this many bytes behind the current one
struct alignas(256) WarpSmem {
  uint64_t ring64[kRing / 8];      // output byte at absolute position x lives at byte x & (kRing-1)
  uint8_t J[kLevels][kWin];
  // The compressed stream reaches shared memory by asynchronous bulk copies (cp.async.bulk + mbarrier: one instruction moves the
  // whole region, no registers, no per-lane address arithmetic), double-buffered: while the batches of one window execute, the
  // region the next window must lie in is already on its way.  A window is a byte offset into one of the two buffers.
  alignas(16) uint8_t stage[2][kStage];
  uint64_t bar[2];                 // one mbarrier per buffer
};
constexpr uint32_t kJOff = kRing;                          // byte offsets inside WarpSmem
constexpr uint32_t kStageOff = kRing + kLevels * kWin;
constexpr uint32_t kBarOff = kStageOff + 2 * kStage;
// where the staging buffers stand: which one holds the current window, what the other one was asked to fetch, barrier phases
struct StageState {
  uint32_t phase;                  // bit b = parity the next wait on bar[b] uses
  int cur;                         // buffer of the current window
  bool pf;                         // a copy into buffer cur ^ 1 was issued and not yet waited for
  int pf_start;                    // stream position (relative to the page's first byte, may be < 0) of that buffer's byte 0
  uint32_t pf_bytes;
};

// Tag-byte tables (256 entries each, shared by the CTA).
//   csz : compressed size of the element, 255 = literal with a multi-byte length field (never part of a batch)
//   lut : len (bits 0-6) | offset bits 8-10 of a 1-byte-offset copy, in place (bits 8-10) | is_lit << 16 | long_lit << 17 |
//         (32 - 8 * offset bytes) << 18 (5 bits) | csz << 24
SNP_FN uint32_t elem_csize(uint32_t t) {
  const uint32_t kind = t & 3;
  if (kind == 0) { const uint32_t l = t >> 2; return l < 60 ? l + 2 : 255u; }
  return kind == 1 ? 2u : (kind == 2 ? 3u : 5u);
}
SNP_FN uint32_t elem_lut(uint32_t t) {
  const uint32_t kind = t & 3;
  uint32_t len, hdr, offhi = 0, is_lit = 0, long_lit = 0, msh = 0;
  if (kind == 0) {
    const uint32_t l = t >> 2;
    is_lit = 1; hdr = 1;
    if (l < 60) len = l + 1; else { len = 0; long_lit = 1; }
  } else if (kind == 1) { len = ((t >> 2) & 7) + 4; hdr = 2; offhi = t >> 5; msh = 24; }
  else if (kind == 2) { len = (t >> 2) + 1; hdr = 3; msh = 16; }
  else { len = (t >> 2) + 1; hdr = 5; msh = 0; }
  const uint32_t csz = long_lit ? 0u : hdr + (is_lit ? len : 0u);
  return len | (offhi << 8) | (is_lit << 16) | (long_lit << 17) | (msh << 18) | (csz << 24);
}

SNP_FN uint64_t funnel64(uint64_t lo, uint64_t hi, uint32_t sh_bits) {   // sh_bits in {0, 8, .., 56}
  return (lo >> sh_bits) | ((hi << 1) << (63 - sh_bits));
}
// 8 bytes of read-only input at any alignment
SNP_FN uint64_t ld8_any(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint64_t* q = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
  return funnel64(snp_ldg64(q), snp_ldg64(q + 1), uint32_t(a & 7) * 8);
}
// 8 bytes of this page's earlier OUTPUT at any alignment (written by this warp: coherent loads, never the read-only path)
SNP_FN uint64_t ld8_out(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const uint32_t sh = uint32_t(a & 3) * 8;
  const uint32_t x = snp_ldcg32(q), y = snp_ldcg32(q + 1), z = snp_ldcg32(q + 2);
  return (uint64_t(snp_funnel_r(y, z, sh)) << 32) | snp_funnel_r(x, y, sh);
}
// the same with aligned 64-bit loads: one where p is 8-aligned (value mode: every lane's source has the batch's alignment)
SNP_FN uint64_t ldcg64(const uint64_t* q) {
#ifdef SNP_HAVE_LDCG64
  return snp_ldcg64(q);
#else
  const uint32_t* w = reinterpret_cast<const uint32_t*>(q);
  return uint64_t(snp_ldcg32(w)) | (uint64_t(snp_ldcg32(w + 1)) << 32);
#endif
}
SNP_FN uint64_t ld8_out64(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint64_t* q = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
  if (!(a & 7)) return ldcg64(q);
  return funnel64(ldcg64(q), ldcg64(q + 1), uint32_t(a & 7) * 8);
}
SNP_FN uint8_t* ring_bytes(WarpSmem& sm) { return reinterpret_cast<uint8_t*>(sm.ring64); }
// 8 ring bytes starting at absolute output position x (any alignment, wraps)
SNP_FN uint64_t ring_ld8(const WarpSmem& sm, uint32_t x) {
  const uint32_t w = (x >> 3) & (kRing / 8 - 1);
  return funnel64(sm.ring64[w], sm.ring64[(w + 1) & (kRing / 8 - 1)], (x & 7) * 8);
}
// 8 bytes at byte address a of the warp's shared block (ring ... window), no ring wrap: a + 8 <= kRing, or inside the staged window
SNP_FN uint64_t sm_ld8(const WarpSmem& sm, uint32_t a) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(&sm) + (a >> 2);
  const uint32_t sh = (a & 3) * 8;
  const uint32_t x = w[0], y = w[1], z = w[2];
  return (uint64_t(snp_funnel_r(y, z, sh)) << 32) | snp_funnel_r(x, y, sh);
}
SNP_FN uint64_t shfl64(uint64_t v, int src) {
  const uint32_t lo = snp_shfl(uint32_t(v), src);
  const uint32_t hi = snp_shfl(uint32_t(v >> 32), src);
  return (uint64_t(hi) << 32) | lo;
}
// byte i (compile-time) of a 32-bit word, zero-extended / the low byte of v placed into byte i of acc
template <int I> SNP_FN uint32_t byte_of(uint32_t x) { return snp_byte_perm(x, 0u, 0x4440u + I); }
template <int I> SNP_FN uint32_t put_byte(uint32_t acc, uint32_t v) {
  return snp_byte_perm(acc, v, I == 0 ? 0x3214u : (I == 1 ? 0x3240u : (I == 2 ? 0x3410u : 0x4210u)));
}

// J[LV][byte I of packed]; smbase = shared-space address of the warp's block (device only)
// store the low `len` (1..8) bytes of w at ring byte rb (no wrap inside the element)
#ifdef __CUDACC__
template <int I, int LV> SNP_FN uint32_t jt_get(const WarpSmem&, uint32_t smbase, uint32_t packed) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1+%2];" : "=r"(v) : "r"(__byte_perm(packed, smbase, 0x7650u + I)), "n"(kJOff + LV * kWin));
  return v;
}
SNP_FN uint32_t sm_base(const WarpSmem& sm) { return uint32_t(__cvta_generic_to_shared(&sm)); }
#define SNP_ST_BYTE(i, v) asm volatile("{ .reg .pred p; setp.gt.u32 p, %2, " #i "; @p st.shared.u8 [%0+" #i "], %1; }" ::"r"(a), "r"(v), "r"(len) : "memory")
SNP_FN void store_elem(WarpSmem&, uint32_t smbase, uint32_t rb, uint64_t w, uint32_t len) {
  const uint32_t a = smbase + rb, lo = uint32_t(w), hi = uint32_t(w >> 32);
  asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(lo) : "memory");
  SNP_ST_BYTE(1, lo >> 8); SNP_ST_BYTE(2, lo >> 16); SNP_ST_BYTE(3, lo >> 24);
  SNP_ST_BYTE(4, hi); SNP_ST_BYTE(5, hi >> 8); SNP_ST_BYTE(6, hi >> 16); SNP_ST_BYTE(7, hi >> 24);
}
#undef SNP_ST_BYTE
#else
template <int I, int LV> SNP_FN uint32_t jt_get(const WarpSmem& sm, uint32_t, uint32_t packed) { return sm.J[LV][(packed >> (8 * I)) & 0xffu]; }
SNP_FN uint32_t sm_base(const WarpSmem&) { return 0; }
SNP_FN void store_elem(WarpSmem& sm, uint32_t, uint32_t rb, uint64_t w, uint32_t len) {
  for (uint32_t i = 0; i < len; i++) reinterpret_cast<uint8_t*>(sm.ring64)[rb + i] = uint8_t(w >> (8 * i));
}
#endif
// bulk_init: once per warp (lane 0 initialises both barriers);  bulk_issue: lane 0 starts the copy of `bytes` (multiple of 16) from the
// 16-byte aligned global address g into buffer b;  bulk_wait: every lane blocks until the copy into buffer b has landed.
#ifdef __CUDACC__
SNP_FN void bulk_init(WarpSmem& sm, int lane) {
  if (lane == 0) {
    const uint32_t a = sm_base(sm) + kBarOff;
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(a) : "memory");
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(a + 8) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  snp_syncwarp();
}
SNP_FN void bulk_issue(WarpSmem& sm, int b, const uint8_t* g, uint32_t bytes, int lane) {
  if (lane == 0) {
    const uint32_t bar = sm_base(sm) + kBarOff + 8u * uint32_t(b), dst = sm_base(sm) + kStageOff + uint32_t(kStage) * uint32_t(b);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // the lanes' earlier reads of this buffer are done (syncwarp before)
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(g), "r"(bytes), "r"(bar) : "memory");
  }
}
SNP_FN void bulk_wait(WarpSmem& sm, int b, uint32_t parity) {
  const uint32_t bar = sm_base(sm) + kBarOff + 8u * uint32_t(b);
  uint32_t done;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  } while (!done);
}
#else
SNP_FN void bulk_init(WarpSmem&, int) {}
SNP_FN void bulk_issue(WarpSmem& sm, int b, const uint8_t* g, uint32_t bytes, int lane) {
  if (lane == 0) for (uint32_t i = 0; i < bytes; i++) sm.stage[b][i] = g[i];
}
SNP_FN void bulk_wait(WarpSmem&, int, uint32_t) { snp_syncwarp(); }
#endif
// start fetching the region that holds stream positions [from, from + kStage) (clamped to the stream's end n) into buffer b
SNP_FN void stage_fetch(WarpSmem& sm, StageState& st, int b, const uint8_t* src, uint32_t n, uint32_t from, int lane) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(src + from) & ~uintptr_t(15);
  const uintptr_t end = (reinterpret_cast<uintptr_t>(src + n) + 15) & ~uintptr_t(15);
  uint32_t bytes = uint32_t(end - a);
  if (bytes > uint32_t(kStage)) bytes = uint32_t(kStage);
  st.pf_start = int(intptr_t(a) - intptr_t(reinterpret_cast<uintptr_t>(src)));
  st.pf_bytes = bytes;
  bulk_issue(sm, b, reinterpret_cast<const uint8_t*>(a), bytes, lane);
}

template <int LV> SNP_FN void jt_level(WarpSmem& sm, uint32_t smbase, uint32_t& jlo, uint32_t& jhi, int lane) {
  uint32_t nlo = 0, nhi = 0;
  nlo = put_byte<0>(nlo, jt_get<0, LV - 1>(sm, smbase, jlo)); nhi = put_byte<0>(nhi, jt_get<0, LV - 1>(sm, smbase, jhi));
  nlo = put_byte<1>(nlo, jt_get<1, LV - 1>(sm, smbase, jlo)); nhi = put_byte<1>(nhi, jt_get<1, LV - 1>(sm, smbase, jhi));
  nlo = put_byte<2>(nlo, jt_get<2, LV - 1>(sm, smbase, jlo)); nhi = put_byte<2>(nhi, jt_get<2, LV - 1>(sm, smbase, jhi));
  nlo = put_byte<3>(nlo, jt_get<3, LV - 1>(sm, smbase, jlo)); nhi = put_byte<3>(nhi, jt_get<3, LV - 1>(sm, smbase, jhi));
  jlo = nlo; jhi = nhi;
  reinterpret_cast<uint2*>(sm.J[LV])[lane] = make_uint2(jlo, jhi);
  snp_syncwarp();
}

// plain copy global->global spread over the warp (source is read-only input)
SNP_FN void warp_copy_in(uint8_t* dst, const uint8_t* src, uint32_t len, int lane) {
  uint32_t head = uint32_t((8 - (reinterpret_cast<uintptr_t>(dst) & 7)) & 7);
  if (head > len) head = len;
  if (uint32_t(lane) < head) dst[lane] = snp_ldg8(src + lane);
  const uint32_t nwords = (len - head) >> 3;
  uint64_t* d8 = reinterpret_cast<uint64_t*>(dst + head);
  const uint8_t* s = src + head;
#pragma unroll 4
  for (uint32_t w = lane; w < nwords; w += 32) d8[w] = ld8_any(s + (size_t(w) << 3));
  const uint32_t done = head + (nwords << 3);
  for (uint32_t i = done + lane; i < len; i += 32) dst[i] = snp_ldg8(src + i);
}

// byte at absolute output position x (< o, i.e. produced by an earlier batch): ring if recent enough, else global
SNP_FN uint8_t old_byte(WarpSmem& sm, const uint8_t* dst, uint32_t o, uint32_t x) {
  return (o - x <= uint32_t(kHist)) ? ring_bytes(sm)[x & (kRing - 1)] : snp_ldcg8(dst + x);
}

// ring -> global in whole 32-byte sectors [fl, align_down(upto, 32)), one 8-byte word per lane and trip; returns the new flush
// position.  (Partial sectors would make L2 fetch the rest of the sector from DRAM before the write-back.)
SNP_FN uint32_t flush_words(const WarpSmem& sm, uint8_t* dst, uint32_t fl, uint32_t upto, int lane) {
  const uint32_t w0 = fl >> 3, w1 = (upto >> 5) << 2;
  uint64_t* d8 = reinterpret_cast<uint64_t*>(dst);
  for (uint32_t w = w0 + lane; w < w1; w += 32) d8[w] = sm.ring64[w & (kRing / 8 - 1)];
  return w1 << 3;
}

// The window that starts at stream position pos, in shared memory: already fetched (or on its way) if the last window's look-ahead
// covers [pos, pos + need), else fetched now; the region of the next window starts on its way into the buffer just left.  Returns the
// byte offset of window position 0 inside the warp's shared block.
SNP_FN uint32_t stage_window(WarpSmem& sm, StageState& st, const uint8_t* src, uint32_t n, uint32_t pos, int lane) {
  const uint32_t avail = n - pos;
  const uint32_t need = avail < uint32_t(kWin + kWinPad) ? avail : uint32_t(kWin + kWinPad);
  const int nb = st.cur ^ 1;
  bool hit = false;
  if (st.pf) {
    bulk_wait(sm, nb, (st.phase >> nb) & 1u);
    st.phase ^= 1u << nb;
    st.pf = false;
    hit = int(pos) >= st.pf_start && pos + need <= uint32_t(st.pf_start + int(st.pf_bytes));
    SNP_STAT(stage_hits, hit ? 1 : 0);
  }
  if (!hit) {
    stage_fetch(sm, st, nb, src, n, pos, lane);
    bulk_wait(sm, nb, (st.phase >> nb) & 1u);
    st.phase ^= 1u << nb;
  }
  const uint32_t wbase = kStageOff + uint32_t(kStage) * uint32_t(nb) + uint32_t(int(pos) - st.pf_start);
  st.cur = nb;
  // look ahead: the next window starts in (pos + kAhead, pos + kWin + 61]; its region goes into the buffer just left
  if (pos + kAhead < n) { stage_fetch(sm, st, nb ^ 1, src, n, pos + kAhead, lane); st.pf = true; }
  return wbase;
}

// The jump tables of the window at wbase (avail stream bytes from its start).  Lane l owns the 8 positions [8l, 8l+8): their tag bytes
// are the window word it just loaded.  J[lv][p] = start of the 2^lv-th element after the one at p, kExit when that leaves the window.
// Positions behind the end of the stream are staged as long-literal tags (csz 255): every chain ends there, and a lookup that lands on
// one finds an element that can never be part of a batch.  csz[...] + p saturates at kExit, so J[lv][kExit] == kExit on every level
// and the lookups need no test.  J32 (level 5) only with vmode.
SNP_FN void build_jump_tables(WarpSmem& sm, uint32_t smbase, uint32_t wbase, uint32_t avail, const uint8_t* __restrict__ csz, bool vmode,
                              int lane) {
  uint32_t jlo, jhi;
  {
    uint64_t w = kFill;
    const int nv = int(avail) - lane * 8;                       // stream bytes in this lane's word
    if (nv > 0) {
      w = sm_ld8(sm, wbase + uint32_t(lane) * 8);
      if (nv < 8) w = (w & ((1ull << (8 * nv)) - 1)) | (kFill << (8 * nv));
    }
    const uint32_t wl = uint32_t(w), wh = uint32_t(w >> 32), p0 = uint32_t(lane) * 8;
    uint32_t a;
    jlo = 0; jhi = 0;
    a = p0 + 0 + csz[byte_of<0>(wl)]; jlo = put_byte<0>(jlo, a < kExit ? a : kExit);
    a = p0 + 1 + csz[byte_of<1>(wl)]; jlo = put_byte<1>(jlo, a < kExit ? a : kExit);
    a = p0 + 2 + csz[byte_of<2>(wl)]; jlo = put_byte<2>(jlo, a < kExit ? a : kExit);
    a = p0 + 3 + csz[byte_of<3>(wl)]; jlo = put_byte<3>(jlo, a < kExit ? a : kExit);
    a = p0 + 4 + csz[byte_of<0>(wh)]; jhi = put_byte<0>(jhi, a < kExit ? a : kExit);
    a = p0 + 5 + csz[byte_of<1>(wh)]; jhi = put_byte<1>(jhi, a < kExit ? a : kExit);
    a = p0 + 6 + csz[byte_of<2>(wh)]; jhi = put_byte<2>(jhi, a < kExit ? a : kExit);
    a = p0 + 7 + csz[byte_of<3>(wh)]; jhi = put_byte<3>(jhi, a < kExit ? a : kExit);
    reinterpret_cast<uint2*>(sm.J[0])[lane] = make_uint2(jlo, jhi);
  }
  snp_syncwarp();
  jt_level<1>(sm, smbase, jlo, jhi, lane);
  jt_level<2>(sm, smbase, jlo, jhi, lane);
  jt_level<3>(sm, smbase, jlo, jhi, lane);
  jt_level<4>(sm, smbase, jlo, jhi, lane);
  if (vmode) jt_level<5>(sm, smbase, jlo, jhi, lane);
}

// stop_at: the consumer only needs the first stop_at bytes of the page (>= ulen: all of it).  Decoding may overshoot by one batch.
// csz / lut: the CTA-shared tag tables (elem_csize / elem_lut).  vmode: try value mode (the page holds 8-byte values; the output is
// right whatever the bytes are, the flag only saves the attempts on pages where it cannot pay).
SNP_FN void snappy_page_body(const uint8_t* __restrict__ src, uint32_t n, uint8_t* __restrict__ dst, uint32_t ulen_expected, uint32_t stop_at,
                             bool vmode, WarpSmem& sm, StageState& st, const uint8_t* __restrict__ csz, const uint32_t* __restrict__ lut,
                             int lane, int* err) {
  uint32_t pos = 0, ulen = 0;
  for (int sh = 0; pos < n && sh < 35; sh += 7) {
    const uint32_t b = snp_ldg8(src + pos++);
    ulen |= (b & 0x7f) << sh;
    if (!(b & 0x80)) break;
  }
  if (ulen != ulen_expected) { if (lane == 0) snp_set_err(err, 101); return; }
  uint8_t* const ring = ring_bytes(sm);
  const uint32_t* const sm32 = reinterpret_cast<const uint32_t*>(&sm);
  const uint8_t* const sm8 = reinterpret_cast<const uint8_t*>(&sm);
  const uint32_t smbase = sm_base(sm);
  uint32_t o = 0;                 // bytes produced so far
  uint32_t fl = 0;                // output bytes [0, fl) are in global memory (fl is a multiple of 32, fl <= o)
  while (pos < n && o < stop_at) {
    const uint32_t avail = n - pos;
    // ---- stage the window (every look at the compressed stream goes through the staged bytes, never a dependent global load)
    snp_syncwarp();
    SNP_STAT(windows, 1);
    const uint32_t wbase = stage_window(sm, st, src, n, pos, lane);
    const uint32_t tag0 = sm8[wbase];
    // ---- literal with an explicit length field: straight copy
    if ((tag0 & 3) == 0 && (tag0 >> 2) >= 60) {
      const uint32_t nb = (tag0 >> 2) - 59;
      uint32_t len = 0;
      for (uint32_t i = 0; i < nb && i + 1 < avail; i++) len |= uint32_t(sm8[wbase + 1 + i]) << (8 * i);
      len += 1;
      if (1 + nb > avail || o + len > ulen || len < 1) { if (lane == 0) snp_set_err(err, 102); return; }
      if (len > avail - 1 - nb) {
        // the literal runs past the end of the stream: an error, unless the stream is a compressed PREFIX (transient loads ship only
        // what a partial decode needs) and the bytes that are there reach the position the consumer stops at
        if (o + (avail - 1 - nb) < stop_at) { if (lane == 0) snp_set_err(err, 102); return; }
        len = avail - 1 - nb;
      }
      const uint8_t* lsrc = src + pos + 1 + nb;
      snp_syncwarp();
      fl = flush_words(sm, dst, fl, o, lane);
      if (uint32_t(lane) < o - fl) dst[fl + lane] = ring[(fl + lane) & (kRing - 1)];     // pending partial sector (< 32 bytes)
      warp_copy_in(dst + o, lsrc, len, lane);
      snp_syncwarp();                                  // every lane has read its pending ring words before the tail below overwrites them
      // the ring keeps the tail of the literal (whole words where possible)
      const uint32_t keep = len < uint32_t(kHist) ? len : uint32_t(kHist);
      const uint32_t k0 = o + len - keep, k1 = o + len;
      const uint32_t a0 = (k0 + 7) & ~7u, a1 = k1 & ~7u;
      if (a0 < a1) {
        for (uint32_t w = (a0 >> 3) + lane; w < (a1 >> 3); w += 32) sm.ring64[w & (kRing / 8 - 1)] = ld8_any(lsrc + ((w << 3) - o));
        if (k0 + lane < a0) ring[(k0 + lane) & (kRing - 1)] = snp_ldg8(lsrc + (k0 + lane - o));
        if (a1 + lane < k1) ring[(a1 + lane) & (kRing - 1)] = snp_ldg8(lsrc + (a1 + lane - o));
      } else {
        for (uint32_t i = k0 + lane; i < k1; i += 32) ring[i & (kRing - 1)] = snp_ldg8(lsrc + (i - o));
      }
      snp_syncwarp();
      pos += 1 + nb + len;
      o += len;
      fl = o & ~31u;
      continue;
    }
    build_jump_tables(sm, smbase, wbase, avail, csz, vmode, lane);
    uint32_t qs = 0;                                   // window-relative start of the next batch
    bool first = true;
    for (;;) {
      if (vmode) {
        // ---------------- value mode: lane k takes the k-th (literal, copy) pair after qs
        uint32_t qv = qs;
#pragma unroll
        for (int lv = 0; lv < 5; lv++)
          if ((lane >> lv) & 1) qv = sm.J[lv + 1][qv];
        const uint32_t el = lut[sm8[wbase + qv]];
        const uint32_t L = el & 0x7fu, lcsz = el >> 24;
        const uint32_t qc = qv + (lcsz < 5u ? lcsz : 5u);         // the copy's tag (stays inside the staged bytes)
        const uint32_t ec = lut[sm8[wbase + qc]];
        const uint32_t ccsz = ec >> 24;
        uint32_t lit4, off;                                        // literal bytes 0..3, copy offset
        {
          const uint32_t p1 = wbase + qv + 1, p2 = wbase + qc + 1;
          lit4 = snp_funnel_r(sm32[p1 >> 2], sm32[(p1 >> 2) + 1], (p1 & 3) * 8);
          const uint32_t raw = snp_funnel_r(sm32[p2 >> 2], sm32[(p2 >> 2) + 1], (p2 & 3) * 8);
          off = (raw & (0xffffffffu >> ((ec >> 18) & 31u))) | (ec & 0x700u);
        }
        // a pair is: a literal of 1..4 bytes (a longer one would need a copy shorter than Snappy's 4 bytes), a copy that completes
        // the value, an offset of whole values that does not reach before the page, both elements staged, the value inside ulen
        const uint32_t k8 = uint32_t(lane) * 8;
        const bool ok = qv != kExit && ((el >> 16) & 3u) == 1u && L <= 4u && !((ec >> 16) & 1u) && (ec & 0x7fu) == 8u - L &&
                        off != 0 && !(off & 7u) && off <= o + k8 && qc + ccsz <= avail && o + k8 + 8 <= ulen;
        const unsigned okm = snp_ballot(ok);
        const int cv = (okm == 0xffffffffu) ? 32 : (snp_ffs(~okm) - 1);
        if (cv >= kMinValues) {
          const bool in = uint32_t(lane) < uint32_t(cv);
          // the source value: off / 8 lanes back inside the batch (parent), else one read of the ring or of the page's output
          const uint32_t back = off >> 3;
          const bool old = in && back > uint32_t(lane);
          uint64_t w = 0;
          const uint32_t ph = o & 7u;                              // the batch's (and every source value's) alignment
          if (old) {
            const uint32_t x = o + k8 - off;
            if (off - k8 > uint32_t(kHist)) w = ld8_out64(dst + x);
            else w = ph ? ring_ld8(sm, x) : sm.ring64[(x >> 3) & (kRing / 8 - 1)];
            const uint64_t lm = (1ull << (8 * L)) - 1;
            w = (w & ~lm) | (uint64_t(lit4) & lm);
          }
          // pointer jumping over the parent links: s = parent lane | L << 5 | literal bytes 1..3 (bytes >= L zero).  Byte j of a
          // value is the literal byte of the first value along its chain whose literal covers j, else the root's byte j.
          uint32_t s = uint32_t(lane);
          if (in) s = (old ? uint32_t(lane) : uint32_t(lane) - back) | (L << 5) | (lit4 & uint32_t((1ull << (8 * L)) - 1) & 0xffffff00u);
#pragma unroll
          for (int it = 0; it < 5; it++) {
            const uint32_t t = snp_shfl(s, int(s & 31u));
            const uint32_t l1 = (s >> 5) & 7u, l2 = (t >> 5) & 7u;
            const uint32_t mine = uint32_t((1ull << (8 * l1)) - 1);   // bytes < l1
            s = (t & 31u) | ((l1 > l2 ? l1 : l2) << 5) | (((s & mine) | (t & ~mine)) & 0xffffff00u);
          }
          const uint32_t lk = (s >> 5) & 7u;
          const uint64_t root = shfl64(w, int(s & 31u));
          const uint64_t v = (root & (~0ull << (8 * lk))) | (s & 0xffffff00u) | (lit4 & 0xffu);
          // store: one aligned ring word per lane; at a phase ph != 0 word k is the funnel of values k - 1 and k
          const uint32_t wb = o >> 3;
          if (!ph) {
            if (in) sm.ring64[(wb + uint32_t(lane)) & (kRing / 8 - 1)] = v;
          } else {
            const uint32_t sh = 8 * ph;
            uint64_t prev = (uint64_t(snp_shfl_up(uint32_t(v >> 32), 1)) << 32) | snp_shfl_up(uint32_t(v), 1);
            uint64_t lo = prev >> (64 - sh);
            if (lane == 0) lo = sm.ring64[wb & (kRing / 8 - 1)] & ((1ull << sh) - 1);
            if (in) sm.ring64[(wb + uint32_t(lane)) & (kRing / 8 - 1)] = lo | (v << sh);
            if (lane == cv - 1) sm.ring64[(wb + uint32_t(lane) + 1) & (kRing / 8 - 1)] = v >> (64 - sh);
          }
          snp_syncwarp();
          const uint32_t T = uint32_t(cv) * 8;
          SNP_STAT(steps, 1); SNP_STAT_VALUE(1); SNP_STAT(elements, 2 * cv); SNP_STAT(bytes, T);
          first = false;
          o += T;
          if (o - fl >= kFlushAt) fl = flush_words(sm, dst, fl, o, lane);
          const uint32_t adv = snp_shfl(qc + ccsz, cv - 1);
          if (adv > kRestage || adv >= avail || o >= stop_at) { pos += adv; break; }
          qs = adv;
          snp_syncwarp();
          continue;
        }
      }
      uint32_t q = qs;
#pragma unroll
      for (int lv = 0; lv < 5; lv++)
        if ((lane >> lv) & 1) q = sm.J[lv][q];
      // ---- decode the element at q (branch-free: tag table + the 4 bytes behind the tag)
      const uint32_t e = lut[sm8[wbase + q]];
      uint32_t len = e & 0x7fu;
      uint32_t ecsz = e >> 24;
      bool is_lit = (e >> 16) & 1u;
      uint32_t off;
      {
        const uint32_t p1 = wbase + q + 1;
        const uint32_t raw = snp_funnel_r(sm32[p1 >> 2], sm32[(p1 >> 2) + 1], (p1 & 3) * 8);
        off = is_lit ? 0u : ((raw & (0xffffffffu >> ((e >> 18) & 31u))) | (e & 0x700u));
      }
      // a long literal ends the batch (straight-copy path); a truncated element is caught by m == 0 / the final size check
      const bool valid = q != kExit && !((e >> 17) & 1u) && q + ecsz <= avail;
      const unsigned vm = snp_ballot(valid);
      const int m = (vm == 0xffffffffu) ? 32 : (snp_ffs(~vm) - 1);   // valid lanes form a prefix
      if (m == 0) {
        if (first) { if (lane == 0) snp_set_err(err, 105); return; }
        pos += qs;                                                 // a long literal (or the window's end) starts here: restage
        break;
      }
      first = false;
      if (lane >= m) { len = 0; ecsz = 0; off = 1; is_lit = true; }
      uint32_t inc = len;                                          // inclusive prefix sum of the output lengths
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const uint32_t t = snp_shfl_up(inc, d); if (lane >= d) inc += t; }
      const uint32_t doff = inc - len;
      {
        const bool bad = lane < m && !is_lit && (off == 0 || off > o + doff);
        if (snp_any(bad)) { if (lane == 0) snp_set_err(err, 103); return; }
      }
      const uint32_t len0 = snp_shfl(len, 0);
      int cnt;                                                     // elements executed by this step (a prefix of the batch)
      uint32_t T;                                                  // their output bytes
      if (len0 <= 8) {
        // ---------------- word mode
        // where does this element's data come from?  0 literal bytes in the window, 1 earlier output (ring / global),
        // 2 one earlier element of this batch (parent, byte delta).  Anything else ends the prefix.
        uint32_t skind = 0, spos = 0;
        bool fail = len > 8;
        const uint32_t s0 = doff - off;                            // source start relative to the batch (meaningful for skind 2)
        if (!is_lit && !fail) {
          if (off >= len) {
            if (s0 + len - 1 >= 0x80000000u) { skind = 1; spos = o + s0; }      // ends before the batch starts
            else if (s0 >= 0x80000000u) fail = true;                          // straddles the batch start
            else skind = 2;
          } else {                                                 // self-overlapping (periodic) copy: fine if its pattern is old
            if (doff == 0) { skind = 1; spos = o - off; } else fail = true;
          }
        }
        // issue the loads of the old / literal sources now: the parent search below hides their latency
        uint64_t w = 0;
        if (lane < m && !fail && skind != 2) {
          const uint32_t r = spos & (kRing - 1);
          if (skind == 1 && o - spos > uint32_t(kHist)) w = ld8_out(dst + spos);
          else if (skind == 1 && r > uint32_t(kRing) - 8) w = ring_ld8(sm, spos);
          else w = sm_ld8(sm, skind == 0 ? wbase + q + 1 : r);
          if (skind == 1 && off < len) {                           // periodic: repeat the first `off` bytes
            w &= (off >= 8) ? ~0ull : ((1ull << (8 * off)) - 1);
            for (uint32_t f = off; f < 8; f <<= 1) w |= w << (8 * f);
          }
        }
        // parent = the element that contains byte s0.  Fixed-width columns compress to elements of ~4 bytes (literal + copy per
        // value, offsets that are multiples of the width), so the element off/4 places back is the first guess; pp = parent lane |
        // byte delta << 8
        uint32_t pp = uint32_t(lane);
        bool need = false;
        {
          const int cand = lane - int(off >> 2);
          const uint32_t x = snp_shfl(doff | (len << 16), cand);
          if (skind == 2) {
            const uint32_t d = s0 - (x & 0xffffu);
            if (cand >= 0 && cand < lane && d < 0x10000u && d + len <= (x >> 16)) pp = uint32_t(cand) | (d << 8);
            else need = true;
          }
        }
        if (snp_any(need)) {
          SNP_STAT(parent_searches, 1);
          // general case: binary search over the element starts (register shuffles only)
          int lo = 0;
#pragma unroll
          for (int step = 16; step > 0; step >>= 1) {
            const int cand = lo + step;
            const uint32_t d = snp_shfl(doff, cand & 31);
            if (need && cand < lane && d <= s0) lo = cand;
          }
          const uint32_t pd = snp_shfl(doff, lo), pl = snp_shfl(len, lo);
          if (need) {
            if (lo >= lane || s0 < pd || s0 + len > pd + pl) fail = true;     // not inside ONE earlier element
            else pp = uint32_t(lo) | ((s0 - pd) << 8);
          }
        }
        const unsigned fm = snp_ballot(fail || lane >= m);
        cnt = fm ? snp_ffs(fm) - 1 : 32;                           // >= 1: element 0 has len <= 8 and an old / literal source
        if (vmode) {
          // end the step right before the last value pair that starts in its second half: the next step begins on a value
          // boundary and can take value mode (a step that began off one, e.g. behind the level prefix, would stay off one)
          const uint32_t nx = snp_shfl(len | (uint32_t(!is_lit && off != 0 && !(off & 7u)) << 8), (lane + 1) & 31);
          const bool pair = lane < 31 && is_lit && len <= 4u && nx == (8u - len) + 0x100u;
          const bool cand = pair && 2 * lane >= cnt && lane < cnt;
          const unsigned pm = snp_ballot(cand);
          const unsigned last = snp_ballot(cand && (pm >> lane) == 1u);   // the highest candidate lane, as one bit
          if (last) cnt = snp_ffs(last) - 1;
        }
        if (lane >= cnt) pp = uint32_t(lane);
        // collapse parent chains (parents are always earlier lanes inside the prefix): parent' = parent's parent, delta' = sum
#pragma unroll
        for (int it = 0; it < 5; it++) pp = snp_shfl(pp, int(pp)) + (pp & ~0xffu);      // (the shuffle takes the lane modulo 32)
        {
          const uint64_t wr = shfl64(w, int(pp));
          if (skind == 2) w = wr >> (8 * (pp >> 8));
        }
        T = snp_shfl(inc, cnt - 1);
        if (o + T > ulen) { if (lane == 0) snp_set_err(err, 103); return; }
        if (lane < cnt) {
          const uint32_t rb = (o + doff) & (kRing - 1);
          if (rb <= uint32_t(kRing) - 8) store_elem(sm, smbase, rb, w, len);   // no wrap inside the element
          else {
#pragma unroll
            for (int i = 0; i < 8; i++)
              if (uint32_t(i) < len) ring[(rb + i) & (kRing - 1)] = uint8_t(w >> (8 * i));
          }
        }
      } else {
        // ---------------- run mode: element 0 is long.  A literal goes alone; a copy takes every following copy with the
        // same offset along (one periodic pattern over the union).
        const uint32_t off0 = snp_shfl(off, 0);
        const bool lit0 = snp_shfl(uint32_t(is_lit), 0) != 0;
        if (lit0) cnt = 1;
        else {
          const unsigned brk = snp_ballot(lane >= m || is_lit || off != off0);
          cnt = brk ? snp_ffs(brk) - 1 : 32;
        }
        T = snp_shfl(inc, cnt - 1);
        if (o + T > ulen) { if (lane == 0) snp_set_err(err, 103); return; }
        snp_syncwarp();
        if (lit0) {
          const uint32_t q0 = snp_shfl(q, 0);
          const uint8_t* ls = src + pos + q0 + 1;
          for (uint32_t i = lane; i < T; i += 32) ring[(o + i) & (kRing - 1)] = snp_ldg8(ls + i);
        } else if (off0 == 8 || off0 == 4 || off0 == 2 || off0 == 1) {
          // the pattern as one 64-bit word, phased for 8-aligned absolute positions (off0 divides 8)
          uint64_t pw = ring_ld8(sm, o - off0);
          pw &= (off0 >= 8) ? ~0ull : ((1ull << (8 * off0)) - 1);
          for (uint32_t f = off0; f < 8; f <<= 1) pw |= pw << (8 * f);
          const uint32_t c = (off0 - (o % off0)) % off0;         // (aligned address - o) mod off0
          const uint64_t W = c ? ((pw >> (8 * c)) | (pw << (64 - 8 * c))) : pw;
          const uint32_t a0 = (o + 7) & ~7u, a1 = (o + T) & ~7u;
          if (a0 < a1) {
            for (uint32_t wd = (a0 >> 3) + lane; wd < (a1 >> 3); wd += 32) sm.ring64[wd & (kRing / 8 - 1)] = W;
            if (o + lane < a0) ring[(o + lane) & (kRing - 1)] = uint8_t(W >> (8 * ((o + lane) & 7)));
            if (a1 + lane < o + T) ring[(a1 + lane) & (kRing - 1)] = uint8_t(W >> (8 * lane));
          } else {
            for (uint32_t i = o + lane; i < o + T; i += 32) ring[i & (kRing - 1)] = uint8_t(W >> (8 * (i & 7)));
          }
        } else {
          // any other offset: byte i of the run = old byte (i mod off0) of the pattern (kept incrementally: no division per byte)
          const uint32_t stride = 32u % off0;
          uint32_t r = uint32_t(lane) % off0;
          for (uint32_t i = lane; i < T; i += 32) {
            const uint32_t x = o - off0 + r;
            ring[(o + i) & (kRing - 1)] = old_byte(sm, dst, o, x);
            r += stride;
            if (r >= off0) r -= off0;
          }
        }
      }
      snp_syncwarp();
      SNP_STAT(steps, 1); SNP_STAT(elements, cnt); SNP_STAT(word_steps, len0 <= 8 ? 1 : 0); SNP_STAT(bytes, T);
      o += T;
      if (o - fl >= kFlushAt) fl = flush_words(sm, dst, fl, o, lane);
      // where the next batch starts: right after the last executed element
      const uint32_t adv = snp_shfl(q + ecsz, cnt - 1);
      if (adv > kRestage || adv >= avail || o >= stop_at) { pos += adv; break; }      // (kRestage + 5 <= kWin: the next header is staged)
      qs = adv;
      snp_syncwarp();
    }
  }
  snp_syncwarp();
  fl = flush_words(sm, dst, fl, o, lane);
  if (fl + lane < o) dst[fl + lane] = ring[(fl + lane) & (kRing - 1)];
  if (o != ulen && o < stop_at) { if (lane == 0) snp_set_err(err, 104); }      // the stream ended before the bytes the consumer needs
}

// One page.  st.phase carries the barriers' phases from page to page; no copy is in flight on return.
SNP_FN void snappy_page(const uint8_t* __restrict__ src, uint32_t n, uint8_t* __restrict__ dst, uint32_t ulen_expected, uint32_t stop_at,
                        WarpSmem& sm, uint32_t& phase, const uint8_t* __restrict__ csz, const uint32_t* __restrict__ lut, int lane, int* err,
                        bool vmode = false) {
  StageState st;
  st.phase = phase; st.cur = 0; st.pf = false; st.pf_start = 0; st.pf_bytes = 0;
  snappy_page_body(src, n, dst, ulen_expected, stop_at, vmode, sm, st, csz, lut, lane, err);
  snp_syncwarp();
  if (st.pf) {                                         // drain the look-ahead nobody came to use
    const int nb = st.cur ^ 1;
    bulk_wait(sm, nb, (st.phase >> nb) & 1u);
    st.phase ^= 1u << nb;
  }
  phase = st.phase;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Gate decoder: the pass bit of every value of a 4-byte column page, straight from its Snappy stream, without producing the page.
// The row-group gate of a gate-first scan needs one bit per row of the gate column, and nothing else reads that column's values, so
// writing the decompressed page only to read it back once cost two page-sized trips through memory per row group.  The parse is the
// byte decoder's (staging, jump tables, tag table: 32 elements per step); execution happens on the values' bits instead of their
// bytes, in a 1 KiB bitmap in shared memory, so a copy from far back reads bits that are still there:
//   * the elements go into a table in shared memory (output start, length, literal position or offset); consecutive copies with one
//     offset are one entry, so a run of a repeated value is one entry whatever its length;
//   * a value inside one literal is tested from the stream bytes;
//   * a value inside one copy whose offset is a multiple of 4 (value-aligned) equals the value `offset / 4` back: the copy's values are
//     the bits of the values before it, repeated with that period; an offset of 1 or 2 has period 4 too, from 4 - offset bytes in;
//   * any other value (bytes from two elements, a copy that is not value-aligned) is resolved byte by byte: each byte follows copy
//     sources through the table back to a literal byte, a periodic run reduced modulo its offset in one step.
// A page this does not fit (a long literal, more entries than the table holds, a byte chase over its hop budget, more rows than the
// bitmap holds, a level prefix that is not all-valid, a damaged stream) returns false before anything is written; the caller decodes it
// the byte way, which reports the same errors as always.
constexpr int kGateCap = 256;      // element-table entries (the bench's tag pages need about 40: 525 elements, runs of one offset merged)
constexpr int kGateRows = 8192;    // rows of the pass bitmap
constexpr int kGateHops = 16;      // copy sources followed to resolve one byte
constexpr uint32_t kGateLit = 0x80000000u;
#ifdef __CUDACC__
#define SNP_POPC(x) __popc(x)
#define SNP_CLZ(x) __clz(x)
#else
#define SNP_POPC(x) __builtin_popcount(x)
#define SNP_CLZ(x) __builtin_clz(x)
#endif
struct GateTab {                   // lives in WarpSmem::ring64: this path never runs the byte executor
  uint32_t d[kGateCap];            // first output byte of the entry
  uint32_t len[kGateCap];          // its output bytes
  uint32_t src[kGateCap];          // literal: kGateLit | stream position of its first byte;  copy: offset
  uint32_t bits[kGateRows / 32];   // bit r & 31 of word r >> 5: value r passes
};
static_assert(sizeof(GateTab) <= sizeof(WarpSmem::ring64), "the gate decoder's tables live in the ring");
// the gate: key = value ^ flip, pass <=> key - lo <= span (32-bit arithmetic), the test of gate_rg_kernel
struct GateTest { uint32_t flip, lo, span; };
SNP_FN bool gate_pass(const GateTest& g, uint32_t v) { return (v ^ g.flip) - g.lo <= g.span; }

// output byte y resolved through the table to a literal byte of the stream; false: over the hop budget
SNP_FN bool gate_byte(const GateTab& t, uint32_t ntab, const uint8_t* __restrict__ src, uint32_t y, uint32_t& out) {
  for (int h = 0; h < kGateHops; h++) {
    uint32_t i = 0;                                              // the last entry that starts at or before y (d[0] = 0)
    for (uint32_t step = kGateCap / 2; step; step >>= 1)
      if (i + step < ntab && t.d[i + step] <= y) i += step;
    const uint32_t s = t.src[i], d = t.d[i];
    if (s & kGateLit) { out = snp_ldg8(src + (s & ~kGateLit) + (y - d)); return true; }
    y = (y - d >= s) ? d - s + (y - d) % s : y - s;              // a source inside the run itself: its first period
  }
  return false;
}
// bits [r, r + 32) of the bitmap
SNP_FN uint32_t gate_get32(const GateTab& t, uint32_t r) {
  const uint32_t w = r >> 5, sh = r & 31;
  if (!sh) return t.bits[w];
  return snp_funnel_r(t.bits[w], w + 1 < uint32_t(kGateRows / 32) ? t.bits[w + 1] : 0u, sh);
}
// OR the low n (<= 32) bits of m into the bitmap at value v (lane 0)
SNP_FN void gate_or(GateTab& t, uint32_t v, uint32_t m) {
  if (!m) return;
  const uint32_t w = v >> 5, sh = v & 31;
  t.bits[w] |= m << sh;
  if (sh && (m >> (32 - sh))) t.bits[w + 1] |= m >> (32 - sh);
}
// values [va, vb) byte by byte: lanes 4k..4k+3 take the bytes of value va + 8j + k; false (on every lane): over the hop budget
SNP_FN bool gate_resolve(GateTab& t, uint32_t ntab, const uint8_t* __restrict__ src, uint32_t P, uint32_t va, uint32_t vb, const GateTest& g,
                         int lane) {
  bool ok = true;
  for (uint32_t v0 = va; v0 < vb; v0 += 8) {
    const uint32_t v = v0 + uint32_t(lane >> 2);
    uint32_t b = 0;
    if (v < vb && !gate_byte(t, ntab, src, P + 4 * v + uint32_t(lane & 3), b)) ok = false;
    const uint32_t b1 = snp_shfl(b, (lane + 1) & 31), b2 = snp_shfl(b, (lane + 2) & 31), b3 = snp_shfl(b, (lane + 3) & 31);
    const bool pass = v < vb && !(lane & 3) && gate_pass(g, b | (b1 << 8) | (b2 << 16) | (b3 << 24));
    const uint32_t m = snp_ballot(pass);
    uint32_t m8 = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) m8 |= ((m >> (4 * k)) & 1u) << k;
    if (lane == 0) gate_or(t, v0, m8);
    snp_syncwarp();
  }
  return !snp_any(!ok);
}
// values [va, vb) inside the literal entry that starts at output byte d, stream position sp
SNP_FN void gate_literal(GateTab& t, const uint8_t* __restrict__ src, uint32_t P, uint32_t d, uint32_t sp, uint32_t va, uint32_t vb,
                         const GateTest& g, int lane) {
  for (uint32_t v0 = va; v0 < vb; v0 += 32) {
    const uint32_t v = v0 + uint32_t(lane);
    bool pass = false;
    if (v < vb) {
      const uint8_t* p = src + sp + (P + 4 * v - d);
      pass = gate_pass(g, uint32_t(snp_ldg8(p)) | (uint32_t(snp_ldg8(p + 1)) << 8) | (uint32_t(snp_ldg8(p + 2)) << 16) |
                              (uint32_t(snp_ldg8(p + 3)) << 24));
    }
    const uint32_t m = snp_ballot(pass);
    if (lane == 0) gate_or(t, v0, m);
    snp_syncwarp();
  }
}
// bits [va, vb) = the bits [va - p, va) repeated (value v equals value v - p, in order), one bitmap word per lane; va >= p
SNP_FN void gate_fill(GateTab& t, uint32_t va, uint32_t vb, uint32_t p, int lane) {
  for (uint32_t w = (va >> 5) + uint32_t(lane); w < ((vb + 31) >> 5); w += 32) {
    const uint32_t x0 = w * 32 > va ? w * 32 : va, x1 = w * 32 + 32 < vb ? w * 32 + 32 : vb;
    const uint32_t r = (x0 - va) % p;                            // value x copies value va - p + (x - va) mod p
    uint32_t pat;                                                // the source bits of x0, x0 + 1, ..
    if (p >= 32) {
      const uint32_t a = gate_get32(t, va - p + r);
      pat = p - r >= 32 ? a : ((a & ((1u << (p - r)) - 1)) | (gate_get32(t, va - p) << (p - r)));
    } else {
      const uint64_t pm = (1ull << p) - 1, base = gate_get32(t, va - p) & pm;
      uint64_t y = ((base >> r) | (base << (p - r))) & pm;
      for (uint32_t l = p; l < 32; l <<= 1) y |= y << l;
      pat = uint32_t(y);
    }
    const uint32_t n = x1 - x0;
    t.bits[w] |= (n >= 32 ? pat : (pat & ((1u << n) - 1))) << (x0 & 31);
  }
  snp_syncwarp();
}

// The body of snappy_gate_page.  On true: bitmap words [0, (nrows + 31) / 32) are in t.bits, *last = 1 + the last passing row (0: none).
SNP_FN bool snappy_gate_body(const uint8_t* __restrict__ src, uint32_t n, uint32_t ulen_expected, bool optional, uint32_t nrows,
                             const GateTest& g, WarpSmem& sm, StageState& st, const uint8_t* __restrict__ csz,
                             const uint32_t* __restrict__ lut, int lane, uint32_t* last) {
  uint32_t pos = 0, ulen = 0;
  for (int sh = 0; pos < n && sh < 35; sh += 7) {
    const uint32_t b = snp_ldg8(src + pos++);
    ulen |= (b & 0x7f) << sh;
    if (!(b & 0x80)) break;
  }
  if (ulen != ulen_expected || nrows == 0 || nrows > uint32_t(kGateRows)) return false;
  if (!optional && ulen != 4 * nrows) return false;
  GateTab& t = *reinterpret_cast<GateTab*>(sm.ring64);
  const uint32_t nw = (nrows + 31) >> 5;
  for (uint32_t w = uint32_t(lane); w < nw; w += 32) t.bits[w] = 0;
  const uint32_t* const sm32 = reinterpret_cast<const uint32_t*>(&sm);
  const uint8_t* const sm8 = reinterpret_cast<const uint8_t*>(&sm);
  const uint32_t smbase = sm_base(sm);
  uint32_t o = 0;                 // bytes produced so far
  uint32_t ntab = 0;              // table entries
  uint32_t P = optional ? 0xffffffffu : 0u;                      // level prefix bytes (optional pages: [u32 length][levels])
  uint32_t vdone = 0, e = 0;      // values [0, vdone) have their bits; the entry that holds the last byte of value vdone is e or later
  while (pos < n) {
    const uint32_t avail = n - pos;
    snp_syncwarp();
    SNP_STAT(windows, 1);
    const uint32_t wbase = stage_window(sm, st, src, n, pos, lane);
    const uint32_t tag0 = sm8[wbase];
    if ((tag0 & 3) == 0 && (tag0 >> 2) >= 60) return false;     // a long literal: an incompressible page, decoded the byte way
    build_jump_tables(sm, smbase, wbase, avail, csz, false, lane);
    uint32_t qs = 0;
    bool first = true;
    for (;;) {
      uint32_t q = qs;
#pragma unroll
      for (int lv = 0; lv < 5; lv++)
        if ((lane >> lv) & 1) q = sm.J[lv][q];
      const uint32_t el = lut[sm8[wbase + q]];
      uint32_t len = el & 0x7fu, ecsz = el >> 24;
      bool is_lit = (el >> 16) & 1u;
      uint32_t off;
      {
        const uint32_t p1 = wbase + q + 1;
        const uint32_t raw = snp_funnel_r(sm32[p1 >> 2], sm32[(p1 >> 2) + 1], (p1 & 3) * 8);
        off = is_lit ? 0u : ((raw & (0xffffffffu >> ((el >> 18) & 31u))) | (el & 0x700u));
      }
      const bool valid = q != kExit && !((el >> 17) & 1u) && q + ecsz <= avail;
      const unsigned vm = snp_ballot(valid);
      const int m = (vm == 0xffffffffu) ? 32 : (snp_ffs(~vm) - 1);
      if (m == 0) {
        if (first) return false;
        pos += qs;
        break;
      }
      first = false;
      const bool in = lane < m;
      if (!in) { len = 0; ecsz = 0; off = 1; is_lit = true; }
      uint32_t inc = len;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const uint32_t x = snp_shfl_up(inc, d); if (lane >= d) inc += x; }
      const uint32_t doff = inc - len;
      if (snp_any(in && !is_lit && (off == 0 || off > o + doff))) return false;
      const uint32_t T = snp_shfl(inc, m - 1);
      if (o + T > ulen) return false;
      // ---- the batch's elements into the table: an element starts an entry unless it is a copy with the offset of the copy before it
      {
        const bool cp = in && !is_lit;
        const uint32_t pc = snp_shfl_up(uint32_t(cp) | (off << 1), 1);
        bool cont;
        if (lane == 0) cont = cp && ntab > 0 && t.src[ntab - 1] == off;
        else cont = cp && (pc & 1u) && (pc >> 1) == off;
        const unsigned hm = snp_ballot(in && !cont);
        const uint32_t nnew = uint32_t(SNP_POPC(hm));
        if (ntab + nnew > uint32_t(kGateCap)) return false;
        const unsigned above = lane == 31 ? 0u : (hm & ~((2u << lane) - 1u));
        const uint32_t nd = snp_shfl(doff, above ? snp_ffs(above) - 1 : 0);
        const uint32_t end = above ? nd : T;                      // where this lane's entry ends inside the batch
        snp_syncwarp();                                           // every lane has read t.src[ntab - 1]
        if (in && !cont) {
          const uint32_t i = ntab + uint32_t(SNP_POPC(hm & ((1u << lane) - 1u)));
          t.d[i] = o + doff;
          t.len[i] = end - doff;
          t.src[i] = is_lit ? (kGateLit | (pos + q + 1)) : off;
        }
        const uint32_t f = snp_shfl(doff, hm ? snp_ffs(hm) - 1 : 0);
        if (lane == 0 && !(hm & 1u)) t.len[ntab - 1] += hm ? f : T;   // the batch continues the table's last run
        ntab += nnew;
        snp_syncwarp();
      }
      o += T;
      SNP_STAT(steps, 1); SNP_STAT(elements, m); SNP_STAT(bytes, T);
      // ---- the level prefix, once its 4 length bytes exist: all-valid pages only (the value count must fill the page)
      if (P == 0xffffffffu && o >= 4) {
        uint32_t b = 0;
        const bool ok = lane >= 4 || gate_byte(t, ntab, src, uint32_t(lane), b);
        if (snp_any(!ok)) return false;
        const uint32_t lv = snp_shfl(b, 0) | (snp_shfl(b, 1) << 8) | (snp_shfl(b, 2) << 16) | (snp_shfl(b, 3) << 24);
        if (lv > ulen - 4 || ulen - 4 - lv != 4 * nrows) return false;
        P = 4 + lv;
      }
      // ---- bits of the values whose last byte now exists, entry by entry
      if (P != 0xffffffffu && o >= P) {
        uint32_t vend = (o - P) / 4;
        vend = vend < nrows ? vend : nrows;
        while (vdone < vend) {
          const uint32_t D = t.d[e], E = D + t.len[e], s = t.src[e];
          uint32_t vl = E >= P ? (E - P) / 4 : 0;
          vl = vl < vend ? vl : vend;
          if (vl <= vdone) {                                      // the next value ends in a later entry
            if (++e >= ntab) return false;
            continue;
          }
          uint32_t v = vdone;
          if (P + 4 * v < D) {                                   // starts in an earlier entry
            if (!gate_resolve(t, ntab, src, P, v, v + 1, g, lane)) return false;
            v++;
          }
          if (v < vl) {
            if (s & kGateLit) {
              gate_literal(t, src, P, D, s & ~kGateLit, v, vl, g, lane);
            } else if (!(s & 3u) || s == 1u || s == 2u) {
              // value-aligned: period s / 4; offsets 1 and 2 repeat every value from 4 - s bytes into the run
              const uint32_t p = (s & 3u) ? 1u : s >> 2;
              uint32_t u = v;
              while (u < vl && (u < p || ((s & 3u) && P + 4 * u < D + 4 - s))) u++;   // sources before the values, or not periodic yet
              if (u > v && !gate_resolve(t, ntab, src, P, v, u, g, lane)) return false;
              if (u < vl) gate_fill(t, u, vl, p, lane);
            } else if (!gate_resolve(t, ntab, src, P, v, vl, g, lane)) {
              return false;
            }
          }
          vdone = vl;
        }
      }
      const uint32_t adv = snp_shfl(q + ecsz, m - 1);
      if (adv > kRestage || adv >= avail) { pos += adv; break; }
      qs = adv;
      snp_syncwarp();
    }
  }
  if (o != ulen || vdone != nrows) return false;
  snp_syncwarp();
  uint32_t lst = 0;
  for (uint32_t w = uint32_t(lane); w < nw; w += 32)
    if (t.bits[w]) lst = w * 32 + 32 - uint32_t(SNP_CLZ(t.bits[w]));
  for (int d = 16; d > 0; d >>= 1) { const uint32_t x = snp_shfl(lst, (lane + d) & 31); lst = x > lst ? x : lst; }
  *last = lst;
  return true;
}

// One 4-byte gate page in the bit domain (see above).  True: bitmap words [0, (nrows + 31) / 32) are in the warp's GateTab and *last
// is 1 + the last passing row (0: none).  False: the page must be decoded the byte way.  st.phase carries the barriers' phases as in
// snappy_page; no copy is in flight on return.
SNP_FN bool snappy_gate_page(const uint8_t* __restrict__ src, uint32_t n, uint32_t ulen_expected, bool optional, uint32_t nrows,
                             const GateTest& g, WarpSmem& sm, uint32_t& phase, const uint8_t* __restrict__ csz,
                             const uint32_t* __restrict__ lut, int lane, uint32_t* last) {
  StageState st;
  st.phase = phase; st.cur = 0; st.pf = false; st.pf_start = 0; st.pf_bytes = 0;
  const bool ok = snappy_gate_body(src, n, ulen_expected, optional, nrows, g, sm, st, csz, lut, lane, last);
  snp_syncwarp();
  if (st.pf) {
    const int nb = st.cur ^ 1;
    bulk_wait(sm, nb, (st.phase >> nb) & 1u);
    st.phase ^= 1u << nb;
  }
  phase = st.phase;
  return ok;
}
SNP_FN const GateTab& gate_tab(const WarpSmem& sm) { return *reinterpret_cast<const GateTab*>(sm.ring64); }

}  // namespace snp
}  // namespace horae
