// radix_agg.cu — GROUP BY for keys that are NOT a prefix of the sort order (e.g. per-(tag, time bucket) aggregates over
// a stream sorted by (series_id, ts): BASELINE config 4b; the aggregation stage itself is todo!() in the reference,
// metric_engine/src/metric/mod.rs:37-49).  Radix-partitioned: the surviving rows are STABLY sorted by the group key with
// an LSD radix sort (8-bit digits, warp-match ranking), so every group becomes one run whose rows keep their stream order;
// the run-based reducers of kernels.cu then add each group's values sequentially in that order — bit-identical to a
// single-threaded hash aggregation that sees the rows in stream order (the oracle's definition).
#include "kernels.h"

namespace horae {
namespace k {

namespace {

constexpr int kThreads = 256;
constexpr int kRounds = 4;                       // items per thread
constexpr int kTile = kThreads * kRounds;        // 1024 items per block, taken in order

// sort keys of the surviving rows: the group value and the bucket start in order-preserving unsigned form
__global__ void __launch_bounds__(kThreads) group_sort_keys_kernel(AggSpecDev spec, const uint32_t* __restrict__ rows, const uint32_t* d_r,
                                                                  uint64_t* __restrict__ gk, uint64_t* __restrict__ bk, uint32_t* __restrict__ vals) {
  const uint32_t r = *d_r;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < r; i += gridDim.x * kThreads) {
    const uint32_t row = rows ? rows[i] : i;
    vals[i] = row;
    if (gk) gk[i] = order_key(widen(col_raw(spec.group, row), spec.group.type), spec.group.type);
    if (bk) {
      const int64_t ts = int64_t(widen(col_raw(spec.ts, row), spec.ts.type));
      bk[i] = order_key(uint64_t(ts / spec.window_ms * spec.window_ms), T_I64);       // truncating division (types.rs:82-85)
    }
  }
}

// per-block digit counts: counts[digit * nb + block]
__global__ void __launch_bounds__(kThreads) radix_hist_kernel(const uint64_t* __restrict__ keys, const uint32_t* d_n, int shift, uint32_t nb,
                                                             uint32_t* __restrict__ counts) {
  __shared__ uint32_t s_h[256];
  const uint32_t n = *d_n;
  s_h[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t base = blockIdx.x * kTile;
#pragma unroll
  for (int r = 0; r < kRounds; r++) {
    const uint32_t i = base + r * kThreads + threadIdx.x;
    if (i < n) atomicAdd(&s_h[uint32_t(keys[i] >> shift) & 255u], 1u);
  }
  __syncthreads();
  counts[threadIdx.x * nb + blockIdx.x] = s_h[threadIdx.x];
}

// stable scatter: an item's position = scanned count of (its digit, its block) + number of earlier items of the block
// with the same digit (earlier rounds, earlier warps of the round, lower lanes of the warp)
__global__ void __launch_bounds__(kThreads) radix_scatter_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, const uint32_t* d_n,
                                                                int shift, uint32_t nb, const uint32_t* __restrict__ scanned,
                                                                uint64_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out) {
  __shared__ uint32_t s_before[256];             // same-digit items of earlier rounds
  __shared__ uint32_t s_w[kThreads / 32][256];   // per warp of the current round
  const uint32_t n = *d_n;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  s_before[threadIdx.x] = 0;
  const uint32_t base = blockIdx.x * kTile;
  for (int r = 0; r < kRounds; r++) {
#pragma unroll
    for (int x = 0; x < kThreads / 32; x++) s_w[x][threadIdx.x] = 0;
    __syncthreads();
    const uint32_t i = base + r * kThreads + threadIdx.x;
    const bool in = i < n;
    uint64_t key = 0;
    uint32_t val = 0, digit = 256 + lane;          // out-of-range items never match anything
    if (in) { key = keys[i]; val = vals[i]; digit = uint32_t(key >> shift) & 255u; }
    const unsigned peers = __match_any_sync(0xffffffffu, digit);
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    if (in && rank == 0) s_w[w][digit] = __popc(peers);
    __syncthreads();
    uint32_t pos = 0;
    if (in) {
      uint32_t earlier = s_before[digit];
      for (int x = 0; x < w; x++) earlier += s_w[x][digit];
      pos = scanned[digit * nb + blockIdx.x] + earlier + rank;
    }
    __syncthreads();
    {
      uint32_t tot = 0;
#pragma unroll
      for (int x = 0; x < kThreads / 32; x++) tot += s_w[x][threadIdx.x];
      s_before[threadIdx.x] += tot;
    }
    if (in) { keys_out[pos] = key; vals_out[pos] = val; }
    __syncthreads();
  }
}

// write path (sort_batch, storage.rs:244-256): order-preserving key of one primary-key column for the rows perm[0..n)
__global__ void __launch_bounds__(kThreads) column_sort_keys_kernel(ColView col, const uint32_t* __restrict__ perm, uint32_t n, uint64_t* __restrict__ keys) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads)
    keys[i] = order_key(widen(col_raw(col, perm[i]), col.type), col.type);
}
__global__ void __launch_bounds__(kThreads) iota_kernel(uint32_t* p, uint32_t n) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) p[i] = i;
}
__global__ void __launch_bounds__(kThreads) fill_u64_kernel(uint64_t* p, uint64_t v, uint32_t n) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) p[i] = v;
}
// Arrow validity bitmap (bit i of byte i/8, LSB first, starting at bit `offset`) -> one byte per row
__global__ void __launch_bounds__(kThreads) unpack_bitmap_kernel(const uint8_t* __restrict__ bitmap, uint64_t offset, uint32_t n, uint8_t* __restrict__ out) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    const uint64_t b = offset + i;
    out[i] = (bitmap[b >> 3] >> (b & 7)) & 1u;
  }
}

}  // namespace

void column_sort_keys(const Launch& L, ColView col, const uint32_t* perm, uint32_t n, uint64_t* keys) {
  if (!n) return;
  column_sort_keys_kernel<<<grid_for(n, kThreads), kThreads, 0, L.stream>>>(col, perm, n, keys);
  L.tick();
}
void iota_u32(const Launch& L, uint32_t* p, uint32_t n) {
  if (!n) return;
  iota_kernel<<<grid_for(n, kThreads), kThreads, 0, L.stream>>>(p, n);
  L.tick();
}
void fill_u64(const Launch& L, uint64_t* p, uint64_t v, uint32_t n) {
  if (!n) return;
  fill_u64_kernel<<<grid_for(n, kThreads), kThreads, 0, L.stream>>>(p, v, n);
  L.tick();
}
void unpack_bitmap(const Launch& L, const uint8_t* bitmap, uint64_t offset, uint32_t n, uint8_t* out) {
  if (!n) return;
  unpack_bitmap_kernel<<<grid_for(n, kThreads), kThreads, 0, L.stream>>>(bitmap, offset, n, out);
  L.tick();
}

size_t radix_tmp_elems(uint32_t cap) { return size_t(256) * ((size_t(cap) + kTile - 1) / kTile) + 16; }

// Stable LSD radix sort of (key, val) pairs over key bits [0, bits).  Returns 0 if the result is in (keys, vals), 1 if it is
// in (keys_tmp, vals_tmp).  The element count lives on the device (*d_n <= cap).
int radix_sort_pairs(const Launch& L, uint64_t* keys, uint32_t* vals, uint64_t* keys_tmp, uint32_t* vals_tmp, const uint32_t* d_n, uint32_t cap,
                     int bits, uint32_t* counts) {
  if (!cap) return 0;
  const uint32_t nb = (cap + kTile - 1) / kTile;
  int where = 0;
  for (int shift = 0; shift < bits; shift += 8) {
    uint64_t* ki = where ? keys_tmp : keys;
    uint32_t* vi = where ? vals_tmp : vals;
    uint64_t* ko = where ? keys : keys_tmp;
    uint32_t* vo = where ? vals : vals_tmp;
    radix_hist_kernel<<<nb, kThreads, 0, L.stream>>>(ki, d_n, shift, nb, counts);
    L.tick();
    exclusive_scan_u32(L, counts, 256 * nb, nullptr);     // digit-major order = final order of the pass
    radix_scatter_kernel<<<nb, kThreads, 0, L.stream>>>(ki, vi, d_n, shift, nb, counts, ko, vo);
    L.tick();
    where ^= 1;
  }
  return where;
}

void group_sort_keys(const Launch& L, const AggSpecDev& spec, const uint32_t* rows, const uint32_t* d_r, uint32_t cap, uint64_t* gk, uint64_t* bk,
                     uint32_t* vals) {
  if (!cap) return;
  group_sort_keys_kernel<<<grid_for(cap, kThreads), kThreads, 0, L.stream>>>(spec, rows, d_r, gk, bk, vals);
  L.tick();
}

}  // namespace k
}  // namespace horae
