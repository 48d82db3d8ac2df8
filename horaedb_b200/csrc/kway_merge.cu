// kway_merge.cu — single-pass k-way merge of the per-SST sorted streams (S4: SortPreservingMergeExec on (pk..., __seq__),
// read.rs:412-427, 479-480; ties -> lower stream index) fused with the PK-run boundaries of S5/S6 (MergeStream +
// LastValueOperator, read.rs:289-343, operator.rs:39-44).  Replaces log2(k) pairwise merge-path passes over 32-byte
// records (64 B of HBM traffic per record per pass) by ONE pass over 8-byte keys:
//
//   keys      every surviving row gets one order-preserving 64-bit key: the primary key columns and __seq__ rebased to
//             the minima the chunk statistics give (so that their spans fit), and the stream index in the low bits — the
//             total order of SortPreservingMergeExec including its tie-break.  (Schemas whose spans do not fit in 52
//             bits stay on the pairwise passes of kernels.cu.)
//   ranges    8192 evenly spaced keys are sorted by one CTA; every (8192/R)-th is a splitter.  One binary search per
//             (splitter, stream) cuts every stream into R key ranges; a range's first output position is the sum of its
//             cut positions, so ranges are independent and need no exact rank selection.
//   merge     one CTA per range (atomic ticket).  Per round it loads the next B = 4096/k keys of every stream into shared
//             memory, takes as threshold the smallest "last loaded key" among the streams that still have more — every
//             loaded key <= threshold is safe to emit, nothing unloaded can precede it — and merges those with a
//             log2(k)-level pairwise merge tree in shared memory (merge-path per thread).  The low 12 bits of the sorted
//             word carry the key's slot in the round, i.e. its stream and position: no payload array.
//   output    row ids in merged order + the "last row of its primary-key run" flag (compare the key's PK part with the
//             next key's; across rounds and ranges the next key is carried / looked up).
#include "kernels.h"

namespace horae {
namespace k {

namespace {

constexpr int kThreads = 256;
constexpr int kMergeThreads = 512;        // merge CTA: 512 threads x 2 CTAs/SM (64 KB of shared memory each): shorter per-thread merge runs
constexpr int kChunk = 4096;              // keys per round in shared memory (two buffers of 32 KB)
constexpr int kIdxBits = 12;              // log2(kChunk): slot of a key inside its round
constexpr int kSamples = 8192;
constexpr uint64_t kInf = ~0ull;

constexpr uint32_t kKeyChunk = 2048;      // survivors per CTA trip of build_keys64_kernel (8 per thread, coalesced)
// WIDE: every primary-key column and __seq__ are 8-byte integers without a validity vector (the metric schema): no per-row dispatch
template <bool WIDE>
__global__ void __launch_bounds__(kThreads) build_keys64_kernel(PkSet pk, ColView seq, const uint32_t* __restrict__ surv, const uint32_t* d_m,
                                                               const uint32_t* __restrict__ run_start, int k, KeyPack kp,
                                                               uint64_t* __restrict__ keys, int* err) {
  __shared__ uint32_t s_rs[kMaxMergeRuns + 2];
  for (int i = threadIdx.x; i <= k; i += kThreads) s_rs[i] = run_start[i];
  __syncthreads();
  const uint32_t m = *d_m;
  bool bad = false;
  uint64_t flip[MAX_PK];
#pragma unroll
  for (int c = 0; c < MAX_PK; c++) flip[c] = c < pk.n ? order_flip(pk.c[c].type) : 0ull;
  for (uint64_t base = uint64_t(blockIdx.x) * kKeyChunk; base < m; base += uint64_t(gridDim.x) * kKeyChunk) {
    uint32_t s = uint32_t(base) + threadIdx.x;
    int lo = 0, hi = k;                       // stream of survivor s: last f with run_start[f] <= s (searched once, then advanced)
    while (lo + 1 < hi) { int mid = (lo + hi) >> 1; if (s_rs[mid] <= s) lo = mid; else hi = mid; }
#pragma unroll
    for (uint32_t t = 0; t < kKeyChunk / kThreads; t++, s += kThreads) {
      if (s >= m) break;
      while (lo + 1 < k && s_rs[lo + 1] <= s) lo++;
      const uint32_t row = surv ? surv[s] : s;
      uint64_t key = uint64_t(lo);
#pragma unroll
      for (int c = 0; c < MAX_PK; c++) {
        if (c >= pk.n) break;
        // primary keys are 1-, 4- or 8-byte integers (validate_schema), so the key rule's float cases never run here
        const uint64_t v = WIDE ? (reinterpret_cast<const uint64_t*>(pk.c[c].vals)[row] ^ flip[c])
                                : order_key(widen(col_raw(pk.c[c], row), pk.c[c].type), pk.c[c].type);
        if (v < kp.mn[c] || v - kp.mn[c] > kp.span[c]) bad = true;     // outside the chunk statistics: the packed key would be wrong
        key |= (v - kp.mn[c]) << kp.shift[c];
      }
      uint64_t q;                                                       // ASC NULLS FIRST: null sorts before every value
      if (WIDE) q = reinterpret_cast<const uint64_t*>(seq.vals)[row] + 1;
      else { const bool sv = seq.valid == nullptr || seq.valid[row] != 0; q = sv ? col_raw(seq, row) + 1 : 0; }
      if (q < kp.seq_min || q - kp.seq_min > kp.seq_span) bad = true;
      key |= (q - kp.seq_min) << kp.seq_shift;
      keys[s] = key;
    }
  }
  if (bad) atomicExch(err, 120);
}

// One CTA: sample, bitonic sort in shared memory, pick R-1 splitters.
__global__ void __launch_bounds__(1024) kway_splitters_kernel(const uint64_t* __restrict__ keys, const uint32_t* d_m, uint32_t R,
                                                              uint64_t* __restrict__ splitters) {
  extern __shared__ uint64_t s_k[];
  const uint32_t m = *d_m;
  for (uint32_t j = threadIdx.x; j < uint32_t(kSamples); j += 1024)
    s_k[j] = m ? keys[uint32_t((uint64_t(j) * m) / kSamples)] : kInf;
  __syncthreads();
  for (uint32_t size = 2; size <= uint32_t(kSamples); size <<= 1)
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      for (uint32_t t = threadIdx.x; t < uint32_t(kSamples) / 2; t += 1024) {
        const uint32_t i = 2 * t - (t & (stride - 1));      // lower index of the pair
        const uint32_t j = i + stride;
        const bool up = (i & size) == 0;
        const uint64_t a = s_k[i], b = s_k[j];
        if ((a > b) == up) { s_k[i] = b; s_k[j] = a; }
      }
      __syncthreads();
    }
  for (uint32_t r = threadIdx.x + 1; r < R; r += 1024) splitters[r - 1] = s_k[uint32_t((uint64_t(r) * kSamples) / R)];
}

// bounds[r * k + f] = number of keys of stream f that precede range r (r = 0..R)
__global__ void __launch_bounds__(kThreads) kway_bounds_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ run_start, int k,
                                                              const uint64_t* __restrict__ splitters, uint32_t R, uint32_t* __restrict__ bounds, int* err) {
  const uint32_t idx = blockIdx.x * kThreads + threadIdx.x;
  if (idx >= (R + 1) * uint32_t(k)) return;
  const uint32_t r = idx / k, f = idx % k;
  const uint32_t base = run_start[f], n = run_start[f + 1] - base;
  // this range's cut and, for the check below, the cut of the range before it: two binary searches advanced in the same loop, so that
  // their (dependent) loads overlap instead of doubling the kernel's latency
  uint32_t lo = 0, hi = 0, lo2 = 0, hi2 = 0;
  uint64_t key = 0, key2 = 0;
  if (r == R) lo = n;
  else if (r > 0) { hi = n; key = splitters[r - 1]; }
  const bool check = r > 1 && r < R;
  if (check) { hi2 = n; key2 = splitters[r - 2]; }
  while (lo < hi || lo2 < hi2) {
    const bool a1 = lo < hi, a2 = lo2 < hi2;
    const uint32_t m1 = (lo + hi) >> 1, m2 = (lo2 + hi2) >> 1;
    const uint64_t k1 = a1 ? keys[base + m1] : 0, k2 = a2 ? keys[base + m2] : 0;
    if (a1) { if (k1 < key) lo = m1 + 1; else hi = m1; }
    if (a2) { if (k2 < key2) lo2 = m2 + 1; else hi2 = m2; }
  }
  // for a sorted stream the earlier cut can never lie behind this one (splitters ascend).  For an unsorted one (a damaged file) it can;
  // the flag sends kway_bounds_monotone_kernel to work
  if (check && lo2 > lo) atomicExch(err, 121);
  bounds[idx] = lo;
}

// Cuts of a stream never go backwards from one range to the next.  They cannot for a sorted stream; for an unsorted one (a damaged
// file) the binary searches above may disagree, and ranges that overlap or leave holes would leave `order` partly unwritten.
// Error path only: one thread per stream walks its R + 1 cuts (a well-formed call returns at the first line).
__global__ void kway_bounds_monotone_kernel(int k, uint32_t R, uint32_t* __restrict__ bounds, int* err) {
  if (*err == 0) return;                       // (set by kway_bounds_kernel when a cut goes backwards; any earlier error: the call fails anyway)
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= k) return;
  uint32_t prev = 0;
  bool bad = false;
  for (uint32_t r = 0; r <= R; r++) {
    const uint32_t b = bounds[r * k + f];
    if (b < prev) { bounds[r * k + f] = prev; bad = true; } else prev = b;
  }
  if (bad) atomicExch(err, 121);
}

// one level of the shared-memory merge tree: lists of `step` streams each are merged pairwise, src -> dst, same offsets
__device__ __forceinline__ void merge_level(const uint64_t* __restrict__ src, uint64_t* __restrict__ dst, const uint32_t* offs, int k, int step,
                                            uint32_t n, int tid) {
  const uint32_t vt = (n + kMergeThreads - 1) / kMergeThreads;
  uint32_t pos = uint32_t(tid) * vt;
  const uint32_t end = pos + vt < n ? pos + vt : n;
  const int npairs = (k + 2 * step - 1) / (2 * step);
  auto off_at = [&](int i) { return offs[i > k ? k : i]; };
  while (pos < end) {
    int lo = 0, hi = npairs;                  // last pair whose start <= pos
    while (lo + 1 < hi) { int mid = (lo + hi) >> 1; if (off_at(2 * mid * step) <= pos) lo = mid; else hi = mid; }
    const uint32_t a0 = off_at(2 * lo * step), a1 = off_at((2 * lo + 1) * step), b1 = off_at((2 * lo + 2) * step);
    const uint32_t seg_end = end < b1 ? end : b1;
    const uint32_t la = a1 - a0, lb = b1 - a1, diag = pos - a0;
    uint32_t l = diag > lb ? diag - lb : 0, h = diag < la ? diag : la;
    while (l < h) {
      const uint32_t mid = (l + h) >> 1;
      if (src[a0 + mid] <= src[a1 + diag - 1 - mid]) l = mid + 1; else h = mid;
    }
    uint32_t ia = l, ib = diag - l;
    uint64_t va = ia < la ? src[a0 + ia] : kInf, vb = ib < lb ? src[a1 + ib] : kInf;
    for (uint32_t o = pos; o < seg_end; o++) {
      const bool take_a = ib >= lb || (ia < la && va <= vb);
      dst[o] = take_a ? va : vb;
      if (take_a) { ia++; va = ia < la ? src[a0 + ia] : kInf; }
      else { ib++; vb = ib < lb ? src[a1 + ib] : kInf; }
    }
    pos = seg_end;
  }
}

__global__ void __launch_bounds__(kMergeThreads, 2) kway_merge_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ surv,
                                                                const uint32_t* __restrict__ run_start, int k, const uint32_t* __restrict__ bounds,
                                                                uint32_t R, uint32_t pk_shift, unsigned int* ticket,
                                                                uint32_t* __restrict__ order, uint8_t* __restrict__ keep, int* err) {
  extern __shared__ uint64_t s_dyn[];          // two key buffers of kChunk words (64 KB: beyond the static limit)
  uint64_t* const s_a = s_dyn;
  uint64_t* const s_b = s_dyn + kChunk;
  __shared__ uint32_t s_cur[kMaxMergeRuns], s_end[kMaxMergeRuns], s_take[kMaxMergeRuns], s_n[kMaxMergeRuns], s_offs[kMaxMergeRuns + 1], s_rs[kMaxMergeRuns + 1];
  __shared__ uint64_t s_thr, s_carry;
  __shared__ uint32_t s_range, s_out, s_any, s_has_carry;
  const int tid = threadIdx.x;
  // keys per stream and round: the largest power of two with k * B <= kChunk (slot -> stream / position by shift and mask)
  uint32_t logB = 0;
  while ((2u << logB) * uint32_t(k) <= uint32_t(kChunk)) logB++;
  const uint32_t B = 1u << logB;
  int levels = 0;
  while ((1 << levels) < k) levels++;
  for (int i = tid; i <= k; i += kMergeThreads) s_rs[i] = run_start[i];
  for (;;) {
    __syncthreads();
    if (tid == 0) s_range = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t r = s_range;
    if (r >= R) return;
    if (tid < k) {
      s_cur[tid] = bounds[r * k + tid]; s_end[tid] = bounds[(r + 1) * k + tid];
      // a stream that is not sorted (a damaged file: the reader trusts the writer's order, read.rs:412-427) can give cuts that go backwards
      if (s_end[tid] < s_cur[tid]) { s_end[tid] = s_cur[tid]; atomicExch(err, 121); }
    }
    if (tid == 0) { s_has_carry = 0; s_out = 0; }
    __syncthreads();
    if (tid == 0) { uint32_t o = 0; for (int f = 0; f < k; f++) o += s_cur[f]; s_out = o; }
    for (;;) {
      __syncthreads();
      // ---- how much of every stream is loaded this round; threshold = smallest last-loaded key of a stream with more to come
      if (tid == 0) { s_thr = kInf; s_any = 0; }
      __syncthreads();
      if (tid < k) {
        const uint32_t rem = s_end[tid] - s_cur[tid];
        const uint32_t take = rem < B ? rem : B;
        s_take[tid] = take;
        if (rem) atomicOr(&s_any, 1u);
        if (rem > B) atomicMin(reinterpret_cast<unsigned long long*>(&s_thr), (unsigned long long)keys[s_rs[tid] + s_cur[tid] + B - 1]);
      }
      __syncthreads();
      if (!s_any) break;
      for (uint32_t i = tid; i < uint32_t(k) * B; i += kMergeThreads) {
        const uint32_t f = i >> logB, j = i & (B - 1);
        s_a[i] = j < s_take[f] ? keys[s_rs[f] + s_cur[f] + j] : kInf;
      }
      __syncthreads();
      const uint64_t thr = s_thr;
      if (tid < k) {                         // keys of the stream that are <= threshold
        const uint64_t* p = s_a + uint32_t(tid) * B;
        uint32_t lo = 0, hi = s_take[tid];
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (p[mid] <= thr) lo = mid + 1; else hi = mid; }
        s_n[tid] = lo;
      }
      __syncthreads();
      if (tid == 0) { uint32_t o = 0; for (int f = 0; f < k; f++) { s_offs[f] = o; o += s_n[f]; } s_offs[k] = o; }
      __syncthreads();
      const uint32_t n = s_offs[k];
      // sorted streams always advance (the stream that set the threshold gives all B keys); an unsorted one may not: an error, not a hang
      if (n == 0) {
        // the call fails, but what follows the merge in the stream indexes by `order`: hand out the rest of the range unmerged, so
        // that `order` stays a permutation of the survivors
        if (tid == 0) {
          atomicExch(err, 121);
          uint32_t o = 0;
          for (int f = 0; f < k; f++) { s_offs[f] = o; o += s_end[f] - s_cur[f]; }
          if (s_has_carry) keep[s_out - 1] = 1;
          s_has_carry = 0;
        }
        __syncthreads();
        const uint32_t out0 = s_out;
        for (int f = 0; f < k; f++) {
          const uint32_t rem = s_end[f] - s_cur[f];
          for (uint32_t j = tid; j < rem; j += kMergeThreads) {
            const uint32_t sidx = s_rs[f] + s_cur[f] + j;
            order[out0 + s_offs[f] + j] = surv ? surv[sidx] : sidx;
            keep[out0 + s_offs[f] + j] = 1;
          }
        }
        break;
      }
      for (uint32_t i = tid; i < uint32_t(k) * B; i += kMergeThreads) {
        const uint32_t f = i >> logB, j = i & (B - 1);
        if (j < s_n[f]) s_b[s_offs[f] + j] = (s_a[i] << kIdxBits) | i;
      }
      __syncthreads();
      uint64_t* src = s_b;
      uint64_t* dst = s_a;
      for (int lv = 0; lv < levels; lv++) {
        merge_level(src, dst, s_offs, k, 1 << lv, n, tid);
        __syncthreads();
        uint64_t* t = src; src = dst; dst = t;
      }
      // ---- emit: row ids in merged order, "last of its PK run" flags
      const uint32_t out0 = s_out;
      const uint32_t sh = pk_shift + kIdxBits;
      if (tid == 0 && s_has_carry && n) keep[out0 - 1] = (s_carry >> sh) != (src[0] >> sh);
      for (uint32_t j = tid; j < n; j += kMergeThreads) {
        const uint64_t w = src[j];
        const uint32_t slot = uint32_t(w) & (kChunk - 1);
        const uint32_t f = slot >> logB, i = slot & (B - 1);
        const uint32_t s = s_rs[f] + s_cur[f] + i;
        order[out0 + j] = surv ? surv[s] : s;
        if (j + 1 < n) keep[out0 + j] = (w >> sh) != (src[j + 1] >> sh);
      }
      __syncthreads();
      if (tid == 0 && n) { s_carry = src[n - 1]; s_has_carry = 1; s_out = out0 + n; }
      if (tid < k) s_cur[tid] += s_n[tid];
    }
    // ---- the last output of the range: compare with the first key of what follows (the smallest key at the streams' cuts)
    if (tid == 0 && s_has_carry) {
      uint64_t nxt = kInf;
      for (int f = 0; f < k; f++) {
        const uint32_t e = s_end[f];
        if (s_rs[f] + e < s_rs[f + 1]) { const uint64_t v = keys[s_rs[f] + e]; if (v < nxt) nxt = v; }
      }
      const uint32_t sh = pk_shift + kIdxBits;
      keep[s_out - 1] = nxt == kInf ? 1 : ((s_carry >> sh) != ((nxt << kIdxBits) >> sh));
    }
  }
}

}  // namespace

size_t kway_tmp_bytes(uint32_t cap, int k, uint32_t* ranges) {
  uint32_t R = cap / 16384u;
  if (R < 1) R = 1;
  if (R > 4096) R = 4096;
  *ranges = R;
  return size_t(cap) * 8 + 16 + size_t(R) * 8 + size_t(R + 1) * size_t(k) * 4 + 64;
}

void kway_merge(const Launch& L, const PkSet& pk, ColView seq, const uint32_t* surv, const uint32_t* d_m, uint32_t cap, const uint32_t* run_start,
                int k, const KeyPack& kp, void* tmp, unsigned int* ticket, uint32_t* order, uint8_t* keep, int* err) {
  if (!cap) return;
  uint32_t R = 1;
  (void)kway_tmp_bytes(cap, k, &R);
  uint64_t* keys = static_cast<uint64_t*>(tmp);
  uint64_t* splitters = keys + cap + 2;
  uint32_t* bounds = reinterpret_cast<uint32_t*>(splitters + R);
  bool wide = seq.width == 8 && seq.valid == nullptr;
  for (int c = 0; c < pk.n; c++) wide = wide && pk.c[c].width == 8 && (pk.c[c].type == T_U64 || pk.c[c].type == T_I64);
  const int nb = grid_for(cap, kKeyChunk);
  if (wide) build_keys64_kernel<true><<<nb, kThreads, 0, L.stream>>>(pk, seq, surv, d_m, run_start, k, kp, keys, err);
  else build_keys64_kernel<false><<<nb, kThreads, 0, L.stream>>>(pk, seq, surv, d_m, run_start, k, kp, keys, err);
  L.tick();
  cudaFuncSetAttribute(kway_splitters_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSamples * 8);      // per device
  cudaFuncSetAttribute(kway_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kChunk * 8);
  kway_splitters_kernel<<<1, 1024, kSamples * 8, L.stream>>>(keys, d_m, R, splitters);
  L.tick();
  kway_bounds_kernel<<<int(((R + 1) * uint64_t(k) + kThreads - 1) / kThreads), kThreads, 0, L.stream>>>(keys, run_start, k, splitters, R, bounds, err);
  L.tick();
  kway_bounds_monotone_kernel<<<(k + 63) / 64, 64, 0, L.stream>>>(k, R, bounds, err);
  L.tick();
  kway_merge_kernel<<<int(R < kNumSMs * 2u ? R : kNumSMs * 2u), kMergeThreads, 2 * kChunk * 8, L.stream>>>(keys, surv, run_start, k, bounds, R, kp.pk_shift, ticket, order, keep, err);
  L.tick();
}

}  // namespace k
}  // namespace horae
