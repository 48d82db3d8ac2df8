// snappy_gate_emu.cpp — TEST INFRASTRUCTURE.  The gate decoder of horaedb_b200/csrc/snappy_core.h (snappy_gate_page: one pass bit per
// value of a 4-byte column page, straight from its Snappy stream) on the CPU, on the coroutine warp of snappy_emu.cpp.  Built by
// tests/test_snappy_gate_bits_emu.py with g++; nothing in the product links it.
#include "warp_emu.h"

struct uint2 { uint32_t x, y; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }

struct EmuStats { long windows, steps, elements, word_steps, bytes, parent_searches, stage_hits; };
static EmuStats g_stats;
#define SNP_STAT(counter, amount) do { if (emu::lane_id() == 0) g_stats.counter += long(amount); } while (0)
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
#define snp_funnel_r(lo, hi, sh) emu::funnel_r((lo), (hi), (sh))
#define snp_byte_perm(a, b, s) emu::byte_perm((a), (b), (s))
#define snp_ffs(x) __builtin_ffs(int(x))
#define snp_set_err(err, code) (*(err) = (code))
#include "../../horaedb_b200/csrc/snappy_core.h"

namespace {
struct Job {
  const uint8_t* src; uint32_t n, ulen, nrows; bool optional; horae::snp::GateTest g;
  horae::snp::WarpSmem* sm; const uint8_t* csz; const uint32_t* lut; uint32_t* bits; uint32_t last; int taken;
};
Job g_job;
void lane_main() {
  using namespace horae::snp;
  const int lane = emu::W->cur;
  uint32_t phase = 0, last = 0;
  bulk_init(*g_job.sm, lane);
  const bool ok = snappy_gate_page(g_job.src, g_job.n, g_job.ulen, g_job.optional, g_job.nrows, g_job.g, *g_job.sm, phase, g_job.csz,
                                   g_job.lut, lane, &last);
  if (ok) {
    const GateTab& t = gate_tab(*g_job.sm);
    for (uint32_t w = uint32_t(lane); w < (g_job.nrows + 31) / 32; w += 32) g_job.bits[w] = t.bits[w];
    if (lane == 0) { g_job.last = last; g_job.taken = 1; }
  }
  emu::lane_exit();
}
}  // namespace

extern "C" void emu_set_order(int order) { emu::g_order = order; }
extern "C" void emu_stats(long* out7) { std::memcpy(out7, &g_stats, sizeof(g_stats)); std::memset(&g_stats, 0, sizeof(g_stats)); }
// The pass bits of one raw Snappy stream of a 4-byte column page (optional: [u32 length][levels] first) into bits[(nrows + 31) / 32].
// Returns 1 when the page was taken in the bit domain (*last = 1 + the last passing row, 0: none), 0 when it must be decoded the byte
// way (bits untouched), or the emulator's error (a collective the lanes did not all reach, ...).
extern "C" int emu_gate_page(const uint8_t* src, uint32_t n, uint32_t ulen, int optional, uint32_t nrows, uint32_t flip, uint32_t lo,
                             uint32_t span, uint32_t* bits, uint32_t* last, long* collectives) {
  using namespace horae::snp;
  static uint8_t csz[256];
  static uint32_t lut[256];
  for (uint32_t t = 0; t < 256; t++) { csz[t] = uint8_t(elem_csize(t)); lut[t] = elem_lut(t); }
  std::vector<uint8_t> in(size_t(n) + 128, 0);
  std::memcpy(in.data() + 32, src, n);
  WarpSmem* sm = static_cast<WarpSmem*>(aligned_alloc(256, sizeof(WarpSmem)));
  std::memset(sm, 0xa5, sizeof(WarpSmem));
  g_job = Job{in.data() + 32, n, ulen, nrows, optional != 0, GateTest{flip, lo, span}, sm, csz, lut, bits, 0, 0};
  const int werr = emu::run_warp(lane_main, collectives);
  free(sm);
  if (werr) return -werr;
  *last = g_job.last;
  return g_job.taken;
}
