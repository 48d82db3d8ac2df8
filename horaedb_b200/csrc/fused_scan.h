// fused_scan.h — single-pass decode+filter+aggregate fast path (fused_scan.cu).
#pragma once
#include "engine_internal.h"

namespace horae {
namespace fused {
constexpr int NOT_APPLICABLE = -1000;
constexpr int kHot = 4;   // hot columns of the fused kernel: pk0, pk1 and up to two further predicate columns

// The shape of a fused aggregate: the columns the kernel reads (slots), the ones it tests on every row (hot slots) and the interval
// the predicates of each hot slot fold into.  It depends on the schema, the predicates and the spec only, never on a file.
struct FusedShape {
  bool has_group = false, has_ts = false, global_mode = false;
  std::vector<uint32_t> slots;      // schema columns: the primary keys first, then predicate / value columns
  int pslot[MAX_PREDS] = {0};       // slot of predicate i
  int value_slot = -1;
  // hot slots: [0] = pk0 (group key), [1] = pk1 (time), [2..3] = further predicate columns; the last one is the gate of the
  // late-materialising kernel.  Interval [klo, khi] of an order-preserving unsigned key.
  int nhot = 2;
  int hot_slot[kHot] = {0, 1, 0, 0};
  bool hot_pred[kHot] = {false};    // some predicate tests the hot slot
  uint64_t klo[kHot] = {0, 0, 0, 0}, khi[kHot] = {~0ull, ~0ull, ~0ull, ~0ull};
  bool empty_interval = false;      // the conjunction passes no row
  // schema column of the gate: the last hot slot when a predicate tests it, else -1
  int gate_col() const { return hot_pred[nhot - 1] ? int(slots[hot_slot[nhot - 1]]) : -1; }
};
// NOT_APPLICABLE when the call has no fused shape, else HG_OK.  The schema and the predicates must be valid.
int fused_shape(const hg_schema_desc* schema, const hg_predicate* preds, size_t np, const hg_agg_spec* agg, FusedShape* shape);

// Returns NOT_APPLICABLE when the inputs do not satisfy the fast path's preconditions (the general pipeline then
// runs), otherwise an hg_status.
int try_scan_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n, const hg_predicate* preds,
                       size_t np, const hg_agg_spec* agg, AggBuffers* out);

// Data-driven row-group pruning for transient (host-resident) SSTs: evaluates the conjunction of the predicates on ONE
// column over the PLAIN values of n row groups (already on the device) and writes flags[i] = 1 iff some row passes.
// The filter runs before merge/dedup (read.rs:459-480), so a row group without a passing row contributes nothing and
// its other columns never have to cross PCIe.  Launched on the engine's stream.
struct GateRg {
  const uint8_t* vals;       // PLAIN values of the gate column — or, with `prefixed`, the page body [u32 len][levels][values]
  uint32_t nrows, prefixed;  //   (a Snappy page decompressed on the device: the level length is only known there)
};
// first / last = the first and the last row (0-based) that pass; first > last: no row passes.  mask: bit b set = a row of
// block b passes, blocks of gate_block_rows(nrows) consecutive rows (32 blocks cover the row group)
struct GateOut { uint32_t first, last, mask; };
inline __host__ __device__ uint32_t gate_block_rows(uint32_t nrows) { const uint32_t b = (nrows + 31u) / 32u; return b < 32u ? 32u : b; }
int gate_row_groups(hg_engine* e, const GateRg* d_rgs, uint32_t n, uint32_t type, const hg_predicate* preds, size_t np, GateOut* d_out);
}  // namespace fused
}  // namespace horae
