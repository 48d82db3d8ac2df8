// engine_internal.h — internals shared by engine.cu and fused_scan.cu (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/horae_gpu.h"
#include "bloom.h"
#include "device_types.h"
#include "kernels.h"
#include "parquet_meta.hpp"

using namespace horae;

// --------------------------------------------------------------------------------------------------- error plumbing
int set_error(int code, const std::string& msg);   // defined in engine.cu (thread-local message)
#define CU_TRY(expr)                                                                                         \
  do {                                                                                                       \
    cudaError_t _e = (expr);                                                                                 \
    if (_e != cudaSuccess)                                                                                   \
      return set_error(HG_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));                     \
  } while (0)

// HORAE_TRACE set: host-side timing lines on stderr (read once per process)
inline bool trace_on() {
  static const bool on = getenv("HORAE_TRACE") != nullptr;
  return on;
}
using HostClock = std::chrono::steady_clock;
inline double elapsed_us(HostClock::time_point a, HostClock::time_point b) { return std::chrono::duration<double, std::micro>(b - a).count(); }

// the Parquet physical type of a column type, as the GPU writer stores it and as the reader expects it
inline PhysType phys_of(uint32_t t) {
  switch (t) {
    case T_U64: case T_I64: return PT_INT64;
    case T_F32: return PT_FLOAT;
    case T_F64: return PT_DOUBLE;
    case T_BINARY: return PT_BYTE_ARRAY;
    default: return PT_INT32;
  }
}
// bytes of one PLAIN value of a fixed-width physical type
inline uint32_t phys_width(int phys) { return (phys == PT_INT32 || phys == PT_FLOAT) ? 4u : 8u; }
// a column's name; "c<N>" when the schema has none
inline std::string col_name(const hg_schema_desc* s, uint32_t c) { return s->names && s->names[c] ? std::string(s->names[c]) : "c" + std::to_string(c); }
inline const char* arrow_format(uint32_t t) {
  static const char* f[] = {"C", "c", "S", "s", "I", "i", "L", "l", "f", "g", "z"};
  return f[t];
}

// Exception barrier of the C ABI: nothing may unwind across an extern "C" frame (the caller is Rust / C).  Host containers
// (std::vector / std::string / make_unique) can throw bad_alloc; everything else is reported as an internal error.
#define HG_GUARD_BEGIN try {
#define HG_GUARD_END                                                                                              \
  }                                                                                                               \
  catch (const std::bad_alloc&) { return set_error(HG_ERR_OOM, "host allocation failed"); }                      \
  catch (const std::exception& ex) { return set_error(HG_ERR_INTERNAL, std::string("exception: ") + ex.what()); } \
  catch (...) { return set_error(HG_ERR_INTERNAL, "unknown exception"); }

// widen a PLAIN-encoded statistics value to the comparison domain (i64 / u64 / f64 bits)
inline uint64_t widen_stat(const uint8_t raw[8], int phys, uint32_t t) {
  if (phys == PT_INT32) {
    int32_t v;
    std::memcpy(&v, raw, 4);
    switch (t) {
      case T_U8: return uint8_t(v);
      case T_U16: return uint16_t(v);
      case T_U32: return uint32_t(v);
      default: return uint64_t(int64_t(v));
    }
  }
  if (phys == PT_FLOAT) {
    float f;
    std::memcpy(&f, raw, 4);
    double d = f;
    uint64_t v;
    std::memcpy(&v, &d, 8);
    return v;
  }
  uint64_t v;
  std::memcpy(&v, raw, 8);
  return v;
}
// The literal of a predicate on a fixed-width column in its widened domain.  Binary literals are bytes (hg_predicate::in_bytes): every
// caller branches on T_BINARY first, and gets 0 here.
inline uint64_t pred_literal(const hg_predicate& p, uint32_t t) {
  if (t == T_BINARY) return 0;
  if (type_is_float(t)) {
    uint64_t v;
    std::memcpy(&v, &p.f64, 8);
    return v;
  }
  return type_is_signed(t) ? uint64_t(p.i64) : p.u64;
}

// ------------------------------------------------------------------------------------------------------ SST residency
// Per (row group, column) planning facts, precomputed at load time: statistics widened to the comparison domain
// (i64 / u64 / f64 bits) so that planning a scan is a tight loop over plain arrays.
struct RgCol {
  uint64_t mn = 0, mx = 0;
  uint32_t scratch = 0;      // decompression scratch of the chunk
  uint8_t has_minmax = 0, null_all = 0, null_none = 0, snappy = 0, _pad0 = 0;
  uint8_t single_page = 0;   // exactly one V1 PLAIN data page, UNCOMPRESSED or SNAPPY (what the fused scan can address by row)
  uint8_t stored = 0;        // Snappy page whose stream is one or two literals (incompressible data): readable in place
  uint8_t _pad = 0;
  uint32_t bloom_blocks = 0; // usable split-block bloom filter of the chunk: its 32-byte blocks (0 = none, or ignored: see bloom_bitset)
  uint64_t bloom_off = 0;    //   and the file offset of its bitset
};

// Bloom-filter pruning (DataFusion's bloom_filter_on_read over the plan's required_guarantees, read.rs:613): a row group is dropped when
// some `=` / `IN` predicate's column has a filter there and none of the predicate's literals may be in it.  Literals are hashed once,
// as the column stores them (PLAIN physical bytes).
struct BloomLits {
  size_t n = 0;                             // predicates that can use a filter
  uint32_t pred[MAX_PREDS] = {0}, col[MAX_PREDS] = {0}, first[MAX_PREDS + 1] = {0};
  std::vector<uint64_t> h;                  // hashes of predicate k's literals: h[first[k] .. first[k + 1])
};
// The bloom hash of a literal in the column's widened domain (i64 / u64 / f64 bits).  False when the column's physical type cannot
// represent it exactly (u8 = 300, an f64 that is no f32, NaN): such a predicate is left to statistics and never probed.
inline bool bloom_literal_hash(uint64_t lit, uint32_t t, uint64_t* h) {
  const int64_t sv = int64_t(lit);
  switch (t) {
    case T_U8: if (lit > 0xffu) return false; *h = bloom::xxh64_4(uint32_t(lit)); return true;
    case T_U16: if (lit > 0xffffu) return false; *h = bloom::xxh64_4(uint32_t(lit)); return true;
    case T_U32: if (lit > 0xffffffffu) return false; *h = bloom::xxh64_4(uint32_t(lit)); return true;
    case T_I8: if (sv < -128 || sv > 127) return false; *h = bloom::xxh64_4(uint32_t(int32_t(sv))); return true;
    case T_I16: if (sv < -32768 || sv > 32767) return false; *h = bloom::xxh64_4(uint32_t(int32_t(sv))); return true;
    case T_I32: if (sv < INT32_MIN || sv > INT32_MAX) return false; *h = bloom::xxh64_4(uint32_t(int32_t(sv))); return true;
    case T_U64: case T_I64: *h = bloom::xxh64_8(lit); return true;
    case T_F64: {
      double d;
      std::memcpy(&d, &lit, 8);
      if (d != d) return false;
      *h = bloom::xxh64_8(lit);
      return true;
    }
    case T_F32: {
      double d;
      std::memcpy(&d, &lit, 8);
      if (d != d) return false;
      const float f = float(d);
      const double back = f;
      uint64_t bb;
      std::memcpy(&bb, &back, 8);
      if (bb != lit) return false;
      uint32_t fb;
      std::memcpy(&fb, &f, 4);
      *h = bloom::xxh64_4(fb);
      return true;
    }
    default: return false;
  }
}
// (HG_OP_IN_SET never uses a filter: a large set would probe every filter thousands of times for little pruning beyond its statistics.)
inline void bloom_literals(const hg_schema_desc* schema, const hg_predicate* preds, size_t np, BloomLits* out) {
  out->n = 0;
  out->h.clear();
  for (size_t i = 0; i < np && i < size_t(MAX_PREDS); i++) {
    const hg_predicate& p = preds[i];
    if (p.op != HG_OP_EQ && p.op != HG_OP_IN) continue;
    const uint32_t t = schema->types[p.column];
    if (t == T_BINARY) continue;              // Binary chunks keep no filter
    const size_t mark = out->h.size();
    bool ok = true;
    uint64_t h = 0;
    if (p.op == HG_OP_EQ) {
      ok = bloom_literal_hash(pred_literal(p, t), t, &h);
      out->h.push_back(h);
    } else
      for (uint32_t j = 0; j < p.in_count && ok; j++) { ok = bloom_literal_hash(p.in_values[j], t, &h); out->h.push_back(h); }
    if (!ok || (p.op == HG_OP_IN && p.in_count == 0)) { out->h.resize(mark); continue; }
    out->pred[out->n] = uint32_t(i);
    out->col[out->n] = p.column;
    out->first[out->n] = uint32_t(mark);
    out->n++;
    out->first[out->n] = uint32_t(out->h.size());
  }
}
// Host probe of one row group (rc = its RgCol row) against the file bytes in host memory
inline bool bloom_may_match_host(const RgCol* rc, const uint8_t* data, const BloomLits& bl) {
  for (size_t k = 0; k < bl.n; k++) {
    const RgCol& c = rc[bl.col[k]];
    if (!c.bloom_blocks) continue;
    bool any = false;
    for (uint32_t j = bl.first[k]; j < bl.first[k + 1] && !any; j++) any = bloom::may_contain(data + c.bloom_off, c.bloom_blocks, bl.h[j]);
    if (!any) return false;
  }
  return true;
}

// The HG_OP_IN_SET predicates of one call: keys[i] = the order keys (order_key) of predicate i's values, sorted and unique; empty for
// every other operator.  Built once per call; the row-group pruning searches it and the filter stage uploads it.
struct InSets {
  std::vector<uint64_t> keys[MAX_PREDS];
  const uint64_t* dev[MAX_PREDS] = {};   // keys[i] on the device, once the call's filter stage has uploaded them (arena memory)
};
void prepare_in_sets(const hg_schema_desc* schema, const hg_predicate* preds, size_t np, InSets* out);   // engine.cu; preds validated

// pk0 bounds of a set of row groups, folded from their pk0 chunk statistics.  ok = false: some row group gives no usable bound (no
// statistics, or NULLs), so the set cannot take part in a PK-disjointness proof.
struct Pk0Range {
  uint64_t mn = 0, mx = 0;
  bool seen = false, ok = true;
  void add(const RgCol& c0, uint32_t t0) {
    if (!c0.has_minmax || !c0.null_none) { ok = false; return; }
    if (!seen) { mn = c0.mn; mx = c0.mx; seen = true; return; }
    if (cmp_widened(c0.mn, mn, cmp_class(t0)) < 0) mn = c0.mn;
    if (cmp_widened(c0.mx, mx, cmp_class(t0)) > 0) mx = c0.mx;
  }
};
// PK-disjointness of the inputs from one pk0 range per input: true when every range is usable and, ordered by minimum, each maximum lies
// strictly below the next minimum.  *order then holds the inputs in that (stable) order.
inline bool pk0_disjoint(const std::vector<Pk0Range>& r, uint32_t t0, std::vector<size_t>* order) {
  for (const Pk0Range& x : r) if (!x.ok) return false;
  order->resize(r.size());
  for (size_t i = 0; i < r.size(); i++) (*order)[i] = i;
  std::stable_sort(order->begin(), order->end(), [&](size_t a, size_t b) { return cmp_widened(r[a].mn, r[b].mn, cmp_class(t0)) < 0; });
  for (size_t j = 0; j + 1 < r.size(); j++)
    if (cmp_widened(r[(*order)[j]].mx, r[(*order)[j + 1]].mn, cmp_class(t0)) >= 0) return false;
  return true;
}

struct SstResident {
  uint64_t id = 0, size = 0;
  FileMetaData meta;
  std::vector<RgCol> rgcol;      // [rg * ncols + col]
  std::vector<uint32_t> rg_rows;
  std::vector<uint8_t> rg_dead;        // transient loads, one per row group: not kept by the load (statistics, bloom filter or gate column)
  RgCol* d_rgcol = nullptr;      // the same two tables in HBM (device-side pruning of the fused path)
  uint32_t* d_rg_rows = nullptr;
  // per-file planning facts (over ALL row groups of the file)
  uint64_t rows_total = 0;
  bool col_null_none[MAX_COLS] = {false}, col_has_minmax[MAX_COLS] = {false};
  bool col_all_single[MAX_COLS] = {false};       // every chunk: one V1 PLAIN page (any supported codec)
  bool col_any_snappy[MAX_COLS] = {false};
  bool col_snappy_all_stored[MAX_COLS] = {false};  // every Snappy chunk of the column is a stored (literal-only) page
  bool col_snappy_any_stored[MAX_COLS] = {false};  // some Snappy chunk of the column is one
  bool col_any_zstd[MAX_COLS] = {false};           // some chunk of the column is Zstandard-compressed (general pipeline only)
  bool any_zstd = false;
  uint32_t col_max_scratch[MAX_COLS] = {0};      // largest decompression scratch of one chunk of the column
  uint64_t col_comp_bytes[MAX_COLS] = {0};       // compressed bytes of the column (work estimate for the decompressor)
  Pk0Range pk0;                  // over the row groups with rows
  uint64_t group_bound = 0;      // sum over row groups of min(#distinct pk0 possible, rows) + 1
  uint8_t* d_bytes = nullptr;
  PageDev* d_pages = nullptr;
  ChunkDev* d_chunks = nullptr;
  uint64_t device_bytes = 0;
  bool owned = true;             // false: transient copy living in the engine arena
  // every chunk of the column is one PLAIN V1 page without NULLs and without Zstandard: the fused scan and the transient gate read
  // its values by row number
  bool row_addressable(uint32_t c) const { return col_all_single[c] && col_null_none[c] && !col_any_zstd[c]; }
  ~SstResident() {
    if (!owned) return;
    if (d_bytes) cudaFree(d_bytes);
    if (d_pages) cudaFree(d_pages);
    if (d_chunks) cudaFree(d_chunks);
    if (d_rgcol) cudaFree(d_rgcol);
    if (d_rg_rows) cudaFree(d_rg_rows);
  }
};

// Device workspace of one engine: a grow-only arena.  Every per-call temporary is a bump allocation; the most recent
// allocation can be popped (LIFO) so large short-lived scratch does not raise the peak; the arena is reset at the start
// of the next call (results handed out as device pointers stay valid until then).  Steady state = no cudaMalloc at all.
struct Arena {
  struct Chunk { char* base; size_t cap, used; };
#ifdef HORAE_EMULATED_BUILD
  static bool chunk_per_alloc() { static const bool on = getenv("HORAE_EMU_GUARD") != nullptr; return on; }
#endif
  std::vector<Chunk> chunks;
  size_t high_water = 0, in_call = 0;
  void* alloc(size_t bytes) {
#ifdef HORAE_EMULATED_BUILD
    const size_t exact = (bytes + 15) & ~size_t(15);
#endif
    bytes = (bytes + 255) & ~size_t(255);
    if (chunks.empty() || chunks.back().used + bytes > chunks.back().cap) {
      size_t cap = std::max<size_t>(bytes, chunks.empty() ? (size_t(64) << 20) : chunks.back().cap * 2);
#ifdef HORAE_EMULATED_BUILD          // the test-suite's CPU emulation (tests/emu): with HORAE_EMU_GUARD every allocation is its own
      if (chunk_per_alloc()) cap = bytes = exact;   // guarded mapping (16-byte granularity): an overrun between arena neighbours is a fault
#endif
      void* p = nullptr;
      if (cudaMalloc(&p, cap) != cudaSuccess) return nullptr;
      chunks.push_back(Chunk{static_cast<char*>(p), cap, 0});
    }
    Chunk& c = chunks.back();
    void* p = c.base + c.used;
    c.used += bytes;
    in_call += bytes;
    if (in_call > high_water) high_water = in_call;
    return p;
  }
  void free_if_top(void* p, size_t bytes) {
    bytes = (bytes + 255) & ~size_t(255);
    if (chunks.empty()) return;
    Chunk& c = chunks.back();
    if (c.used >= bytes && c.base + c.used - bytes == static_cast<char*>(p)) { c.used -= bytes; in_call -= bytes; }
  }
  // start of a call (stream idle): one chunk big enough for everything seen so far
  void reset() {
    in_call = 0;
#ifdef HORAE_EMULATED_BUILD
    if (chunk_per_alloc()) { destroy(); return; }
#endif
    if (chunks.size() > 1) {
      size_t total = 0;
      for (auto& c : chunks) { total += c.cap; cudaFree(c.base); }
      chunks.clear();
      void* p = nullptr;
      if (cudaMalloc(&p, total) == cudaSuccess) chunks.push_back(Chunk{static_cast<char*>(p), total, 0});
    } else if (!chunks.empty()) chunks[0].used = 0;
  }
  void destroy() {
    for (auto& c : chunks) cudaFree(c.base);
    chunks.clear();
  }
};
extern thread_local Arena* g_arena;   // arena of the engine whose call is running on this thread (engine.cu)

// per-call device buffer (arena-backed)
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; }
  DevBuf& operator=(DevBuf&& o) noexcept { if (this != &o) { reset(); p = o.p; bytes = o.bytes; o.p = nullptr; } return *this; }
  ~DevBuf() { reset(); }
  void reset() {
    if (p && g_arena) g_arena->free_if_top(p, bytes);
    p = nullptr;
  }
  cudaError_t alloc(size_t nbytes, cudaStream_t) {
    reset();
    bytes = nbytes ? nbytes : 16;
    p = g_arena ? g_arena->alloc(bytes) : nullptr;
    return p ? cudaSuccess : cudaErrorMemoryAllocation;
  }
  void* release() { void* q = p; p = nullptr; return q; }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct hg_comm;
void hg_comm_free(hg_comm* c);   // comm.cu

struct hg_engine {
  int device = 0;
  cudaStream_t stream = nullptr;
  uint32_t batch_size = 8192;
  uint32_t flags = 0;
  uint64_t budget = 0;
  std::mutex mu;
  std::unordered_map<uint64_t, std::unique_ptr<SstResident>> ssts;
  uint64_t resident_bytes = 0;
  hg_scan_stats stats{};
  uint32_t launches = 0;
  size_t stage_cursor = 0;             // next free byte of h_stage in the current call
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evk0 = nullptr, evk1 = nullptr, evm0 = nullptr, evm1 = nullptr, evd0 = nullptr, evd1 = nullptr;  // call / dominant-kernel / merge brackets
  void* h_stage = nullptr;       // pinned staging for per-scan descriptor uploads
  size_t h_stage_bytes = 0;
  void* h_small = nullptr;       // 256 pinned bytes: the per-call counter block comes back here (one small D2H)
  Arena arena;
  hg_agg_device last_agg{};      // device pointers of the last aggregate (arena memory, valid until the next call)
  uint32_t last_gwidth = 8, last_gtype = T_U64;
  struct hg_comm* comm = nullptr;  // NCCL communicator + combine stream (comm.cu)
  std::vector<uint64_t> transient_ids;   // SSTs loaded only for the running call
  uint32_t trunc_mask = 0;               // bit c: the running call reads column c of a row group only up to its last gate-passing row
  int trunc_gate = -1;                    // ... and the column whose predicates define that row (the device's gate column)
  bool trunc_used = false;               // the transient load shipped a compressed PREFIX of some page (see add_prefix)
  InSets in_sets;                        // the running call's HG_OP_IN_SET predicates (begin_call)
  Launch L() { return Launch{stream, &launches}; }
};



struct AggBuffers {
  DevBuf gkey, bucket, count, sum, mn, mx;
  uint32_t G = 0;
  uint32_t gwidth = 8, gtype = T_U64;
  // room for n groups in each column (8 bytes a value, plus 16 so that no buffer is empty)
  cudaError_t alloc(uint64_t n, cudaStream_t s) {
    for (DevBuf* b : {&gkey, &bucket, &count, &sum, &mn, &mx}) {
      const cudaError_t rc = b->alloc(size_t(n) * 8 + 16, s);
      if (rc != cudaSuccess) return rc;
    }
    return cudaSuccess;
  }
  AggOut out() const { return AggOut{gkey.p, bucket.as<int64_t>(), count.as<uint64_t>(), sum.as<double>(), mn.as<double>(), mx.as<double>()}; }
};


struct ScanPlan {
  std::vector<SstResident*> files;     // in decode order
  std::vector<RgSel> sel;
  std::vector<uint32_t> file_base;     // decoded-row base per file (k+1)
  std::vector<uint32_t> piece_end;     // single-SST pass-through: reader batch boundaries (decoded rows)
  uint64_t rows_in_files = 0, rows_decoded = 0, scratch_bytes = 0;
  bool disjoint = false;               // concatenation in decode order is sorted by PK with no cross-file equal PKs
  std::vector<bool> col_has_nulls;     // per schema column: may any selected chunk contain nulls?
};


// Copies `bytes` of host data to the device through the engine's pinned staging area (async on the engine stream;
// the staging area is reused by the next call, which is safe because every call ends with a stream synchronise).
int stage_upload(hg_engine* e, void* dst, const void* src, size_t bytes);
