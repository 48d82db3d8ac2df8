// snappy_value_emu.cpp — TEST INFRASTRUCTURE.  The product's warp-level Snappy decoder (horaedb_b200/csrc/snappy_core.h) on the CPU
// with value mode switchable, as snappy_pages_kernel runs it on INT64 / DOUBLE pages: the same coroutine warp as snappy_emu.cpp, plus
// a value-mode step counter and the 64-bit coherent load the GPU build uses.  Built by tests/test_snappy_value_mode_emu.py and
// tools/snappy_page_stats.py with g++; nothing in the product links it.
#include "warp_emu.h"

struct uint2 { uint32_t x, y; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }

// dynamic counters of the decoder's loop (lane 0 counts): windows, steps, elements, word_steps, bytes, parent_searches, stage_hits,
// value_steps (steps counts every step; word_steps and value_steps the ones of those two modes)
struct EmuStats { long windows, steps, elements, word_steps, bytes, parent_searches, stage_hits, value_steps; };
static EmuStats g_stats;
#define SNP_STAT(counter, amount) do { if (emu::lane_id() == 0) g_stats.counter += long(amount); } while (0)
#define SNP_STAT_VALUE(amount) SNP_STAT(value_steps, amount)
#define SNP_FN static inline
#define snp_shfl(v, src) emu::shfl(uint32_t(v), int(src))
#define snp_shfl_up(v, d) emu::shfl_up(uint32_t(v), int(d))
#define snp_ballot(p) emu::ballot(bool(p))
#define snp_any(p) (emu::ballot(bool(p)) != 0)
#define snp_syncwarp() ((void)emu::rendezvous(0))
#define snp_ldg8(p) (*(p))
#define snp_ldg64(p) (*(p))
#define snp_ldcg8(p) (*(p))
#define snp_ldcg32(p) (*(p))
#define SNP_HAVE_LDCG64 1
#define snp_ldcg64(p) (*(p))
#define snp_funnel_r(lo, hi, sh) emu::funnel_r((lo), (hi), (sh))
#define snp_byte_perm(a, b, s) emu::byte_perm((a), (b), (s))
#define snp_ffs(x) __builtin_ffs(int(x))
#define snp_set_err(err, code) (*(err) = (code))
#include "../../horaedb_b200/csrc/snappy_core.h"

namespace {
struct Job {
  const uint8_t* src; uint32_t n; uint8_t* dst; uint32_t ulen, stop_at;
  horae::snp::WarpSmem* sm; const uint8_t* csz; const uint32_t* lut; int* err;
};
Job g_job;
bool g_vmode = true;
void lane_main() {
  const int lane = emu::W->cur;
  uint32_t phase = 0;
  horae::snp::bulk_init(*g_job.sm, lane);
  horae::snp::snappy_page(g_job.src, g_job.n, g_job.dst, g_job.ulen, g_job.stop_at, *g_job.sm, phase, g_job.csz, g_job.lut, lane,
                          g_job.err, g_vmode);
  emu::lane_exit();
}
}  // namespace

extern "C" void emu_set_order(int order) { emu::g_order = order; }
// value mode on (1, the default: INT64 / DOUBLE pages) or off (0: every other page, and the decoder as it was without value mode)
extern "C" void emu_set_value_mode(int on) { g_vmode = on != 0; }
extern "C" void emu_stats(long* out8) { std::memcpy(out8, &g_stats, sizeof(g_stats)); std::memset(&g_stats, 0, sizeof(g_stats)); }
// Decode one raw Snappy stream.  dst must have ulen + 64 bytes of room.  Returns the decoder's error word (0 = ok).
extern "C" int emu_snappy_page(const uint8_t* src, uint32_t n, uint8_t* dst, uint32_t ulen, uint32_t stop_at, long* collectives) {
  using namespace horae::snp;
  static uint8_t csz[256];
  static uint32_t lut[256];
  for (uint32_t t = 0; t < 256; t++) { csz[t] = uint8_t(elem_csize(t)); lut[t] = elem_lut(t); }
  std::vector<uint8_t> in(size_t(n) + 128, 0);       // slack on both sides: the decoder loads aligned words around unaligned addresses
  std::memcpy(in.data() + 32, src, n);
  WarpSmem* sm = static_cast<WarpSmem*>(aligned_alloc(256, sizeof(WarpSmem)));
  std::memset(sm, 0xa5, sizeof(WarpSmem));
  int err = 0;
  g_job = Job{in.data() + 32, n, dst, ulen, stop_at, sm, csz, lut, &err};
  const int werr = emu::run_warp(lane_main, collectives);
  if (werr) err = werr;
  free(sm);
  return err;
}
