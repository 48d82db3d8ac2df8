// comm.cu — multi-GPU combine of the per-GPU partial aggregates, inside the library (SURVEY 8e; north_star: "a single NCCL
// reduce of per-GPU partial aggregates over NVLink").  One engine per GPU / per process; the host only ships the 128-byte
// NCCL id between ranks (hg_comm_unique_id -> its own channel -> hg_comm_init), exactly what a Rust host would do.
//
//   GATHER   group keys contain the series id and every SST belongs to one rank  => partials are disjoint: ONE
//            ncclAllGather of the packed [6][cap] block of every rank.
//   REDUCE   keys that cross ranks (per-(tag, bucket), config 4b): the same all-gather, then every rank combines the
//            world x cap partial rows itself — stable radix sort by (key, bucket) over the rank-major concatenation, then
//            per group: counts summed, min/max taken, f64 sums added IN RANK ORDER (deterministic; the oracle's multi-shard
//            definition) — so all ranks hold the identical table without a second collective.
//
// The collective runs on its own stream: the pack kernel runs on the engine stream right behind the scan, an event hands
// over, and the next scan call overlaps the all-gather.  NCCL is bound at run time (dlopen libnccl.so.2) so that the library
// has no link-time dependency and shares the copy a host process may already have loaded.
#include <dlfcn.h>

#include "block_scan.h"
#include "engine_internal.h"

namespace {

typedef struct { char internal[128]; } nccl_uid;
typedef void* nccl_comm;
struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(nccl_uid*) = nullptr;
  int (*CommInitRank)(nccl_comm*, int, nccl_uid, int) = nullptr;
  int (*CommDestroy)(nccl_comm) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, nccl_comm, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  std::string err;
};
constexpr int kNcclInt64 = 4;

NcclApi* nccl_api() {
  static NcclApi* api = [] {
    auto* a = new NcclApi();
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) { a->handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (a->handle) break; }
    if (!a->handle) { a->err = std::string("cannot load libnccl: ") + dlerror(); return a; }
    a->GetUniqueId = reinterpret_cast<int (*)(nccl_uid*)>(dlsym(a->handle, "ncclGetUniqueId"));
    a->CommInitRank = reinterpret_cast<int (*)(nccl_comm*, int, nccl_uid, int)>(dlsym(a->handle, "ncclCommInitRank"));
    a->CommDestroy = reinterpret_cast<int (*)(nccl_comm)>(dlsym(a->handle, "ncclCommDestroy"));
    a->AllGather = reinterpret_cast<int (*)(const void*, void*, size_t, int, nccl_comm, cudaStream_t)>(dlsym(a->handle, "ncclAllGather"));
    a->GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(a->handle, "ncclGetErrorString"));
    if (!a->GetUniqueId || !a->CommInitRank || !a->CommDestroy || !a->AllGather || !a->GetErrorString) a->err = "libnccl lacks a required symbol";
    return a;
  }();
  return api;
}

#define NCCL_TRY(api, expr)                                                                                 \
  do {                                                                                                      \
    int _r = (expr);                                                                                        \
    if (_r != 0) return set_error(HG_ERR_CUDA, std::string(#expr) + ": " + (api)->GetErrorString(_r));      \
  } while (0)

}  // namespace

struct hg_comm {
  nccl_comm comm = nullptr;
  int rank = 0, world = 1;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_packed = nullptr, ev_done = nullptr;
  uint64_t cap = 0;                     // columns per rank block of the buffers below
  long long* d_send = nullptr;          // [6][cap]
  long long* d_recv = nullptr;          // [world][6][cap]
  unsigned long long* d_sizes = nullptr;   // [world + 1]
  unsigned long long* h_sizes = nullptr;   // pinned
  // REDUCE scratch (world * cap entries)
  uint64_t red_cap = 0;
  uint64_t *d_k1 = nullptr, *d_k2 = nullptr;
  uint32_t *d_v1 = nullptr, *d_v2 = nullptr, *d_counts = nullptr, *d_seg = nullptr, *d_tmp = nullptr, *d_n = nullptr;
  uint8_t* d_head = nullptr;
  long long* d_out = nullptr;           // [6][red_cap]: combined table
  uint32_t launches = 0;
};

namespace {

// entries of the rank-major concatenation that carry a group (count > 0), in order: idx -> vals, bucket key -> keys
__global__ void __launch_bounds__(256) red_collect_kernel(const long long* __restrict__ recv, uint32_t world, uint64_t cap, uint32_t* __restrict__ vals,
                                                          uint32_t* d_n) {
  // one block, ordered compaction (the tables are small: world x cap entries)
  __shared__ uint32_t s_w[256 / 32 + 1];
  const uint64_t total = uint64_t(world) * cap;
  uint32_t base = 0;
  for (uint64_t b = 0; b < total; b += 256) {
    const uint64_t i = b + threadIdx.x;
    uint32_t f = 0;
    if (i < total) { const uint64_t r = i / cap, j = i % cap; f = recv[(r * 6 + 2) * cap + j] != 0; }
    uint32_t n;
    const uint32_t pos = base + block_excl_scan<256>(f, &n, s_w);
    if (f) vals[pos] = uint32_t(i);
    base += n;
  }
  if (threadIdx.x == 0) *d_n = base;
}

__global__ void __launch_bounds__(256) red_keys_kernel(const long long* __restrict__ recv, uint64_t cap, const uint32_t* __restrict__ vals, const uint32_t* d_n,
                                                       int which, uint32_t gtype, uint64_t* __restrict__ keys) {
  const uint32_t n = *d_n;
  for (uint32_t i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
    const uint64_t e = vals[i], r = e / cap, j = e % cap;
    // the bucket is an i64; the group key is the group value at its native width, zero-extended (pack_agg_kernel)
    keys[i] = which == 0 ? order_key(uint64_t(recv[(r * 6 + 1) * cap + j]), T_I64) : order_key(widen(uint64_t(recv[(r * 6 + 0) * cap + j]), gtype), gtype);
  }
}

__global__ void __launch_bounds__(256) red_heads_kernel(const long long* __restrict__ recv, uint64_t cap, const uint32_t* __restrict__ vals, const uint32_t* d_n,
                                                        uint32_t cap_flags, uint8_t* __restrict__ head) {
  const uint32_t n = *d_n;
  for (uint32_t i = blockIdx.x * 256 + threadIdx.x; i < cap_flags; i += gridDim.x * 256) {
    uint8_t h = 0;
    if (i < n) {
      h = i == 0;
      if (!h) {
        const uint64_t a = vals[i - 1], b = vals[i];
        const uint64_t ra = a / cap, ja = a % cap, rb = b / cap, jb = b % cap;
        h = recv[(ra * 6 + 0) * cap + ja] != recv[(rb * 6 + 0) * cap + jb] || recv[(ra * 6 + 1) * cap + ja] != recv[(rb * 6 + 1) * cap + jb];
      }
    }
    head[i] = h;
  }
}

// one thread per combined group: partial rows in sorted (stable => rank) order
__global__ void __launch_bounds__(256) red_reduce_kernel(const long long* __restrict__ recv, uint64_t cap, const uint32_t* __restrict__ vals, const uint32_t* d_n,
                                                         const uint32_t* __restrict__ seg, const uint32_t* d_g, uint64_t out_cap, long long* __restrict__ out) {
  const uint32_t n = *d_n, g_total = *d_g;
  for (uint32_t g = blockIdx.x * 256 + threadIdx.x; g < g_total; g += gridDim.x * 256) {
    const uint32_t lo = seg[g], hi = g + 1 < g_total ? seg[g + 1] : n;
    unsigned long long cnt = 0;
    double sum = 0.0, mn = 0.0, mx = 0.0;
    long long key = 0, bucket = 0;
    for (uint32_t i = lo; i < hi; i++) {
      const uint64_t e = vals[i], r = e / cap, j = e % cap;
      const long long* blk = recv + r * 6 * cap;
      const double s = __longlong_as_double(blk[3 * cap + j]), a = __longlong_as_double(blk[4 * cap + j]), b = __longlong_as_double(blk[5 * cap + j]);
      if (i == lo) { key = blk[j]; bucket = blk[cap + j]; sum = s; mn = a; mx = b; }
      else { sum += s; mn = a < mn ? a : mn; mx = b > mx ? b : mx; }       // rank-ordered add of the partial sums
      cnt += (unsigned long long)blk[2 * cap + j];
    }
    out[g] = key;
    out[out_cap + g] = bucket;
    out[2 * out_cap + g] = (long long)cnt;
    out[3 * out_cap + g] = __double_as_longlong(sum);
    out[4 * out_cap + g] = __double_as_longlong(mn);
    out[5 * out_cap + g] = __double_as_longlong(mx);
  }
}

int ensure_buffers(hg_comm* c, uint64_t cap, bool reduce) {
  if (cap > c->cap) {
    if (c->d_send) cudaFree(c->d_send);
    if (c->d_recv) cudaFree(c->d_recv);
    c->d_send = nullptr; c->d_recv = nullptr;
    CU_TRY(cudaMalloc(&c->d_send, size_t(6) * cap * 8));
    CU_TRY(cudaMalloc(&c->d_recv, size_t(c->world) * 6 * cap * 8));
    c->cap = cap;
  }
  const uint64_t need = uint64_t(c->world) * c->cap;
  if (reduce && need > c->red_cap) {
    for (void* p : {(void*)c->d_k1, (void*)c->d_k2, (void*)c->d_v1, (void*)c->d_v2, (void*)c->d_counts, (void*)c->d_seg, (void*)c->d_tmp, (void*)c->d_head, (void*)c->d_out})
      if (p) cudaFree(p);
    CU_TRY(cudaMalloc(&c->d_k1, need * 8 + 16));
    CU_TRY(cudaMalloc(&c->d_k2, need * 8 + 16));
    CU_TRY(cudaMalloc(&c->d_v1, need * 4 + 16));
    CU_TRY(cudaMalloc(&c->d_v2, need * 4 + 16));
    CU_TRY(cudaMalloc(&c->d_counts, k::radix_tmp_elems(uint32_t(need)) * 4));
    CU_TRY(cudaMalloc(&c->d_seg, need * 4 + 16));
    CU_TRY(cudaMalloc(&c->d_tmp, k::compact_tmp_elems(uint32_t(need)) * 4 + 16));
    CU_TRY(cudaMalloc(&c->d_head, need + 16));
    CU_TRY(cudaMalloc(&c->d_out, need * 6 * 8 + 16));
    c->red_cap = need;
  }
  return HG_OK;
}

}  // namespace

void hg_comm_free(hg_comm* c) {
  if (!c) return;
  if (c->stream) cudaStreamSynchronize(c->stream);
  NcclApi* api = nccl_api();
  if (c->comm && api->CommDestroy) api->CommDestroy(c->comm);
  for (void* p : {(void*)c->d_send, (void*)c->d_recv, (void*)c->d_sizes, (void*)c->d_k1, (void*)c->d_k2, (void*)c->d_v1, (void*)c->d_v2, (void*)c->d_counts,
                  (void*)c->d_seg, (void*)c->d_tmp, (void*)c->d_head, (void*)c->d_out, (void*)c->d_n})
    if (p) cudaFree(p);
  if (c->h_sizes) cudaFreeHost(c->h_sizes);
  if (c->ev_packed) cudaEventDestroy(c->ev_packed);
  if (c->ev_done) cudaEventDestroy(c->ev_done);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

extern "C" {

int hg_comm_unique_id(uint8_t* id) {
  HG_GUARD_BEGIN
  if (!id) return set_error(HG_ERR_INVALID, "null argument");
  NcclApi* api = nccl_api();
  if (!api->err.empty()) return set_error(HG_ERR_UNSUPPORTED, api->err);
  nccl_uid u;
  NCCL_TRY(api, api->GetUniqueId(&u));
  std::memcpy(id, u.internal, HG_COMM_ID_BYTES);
  return HG_OK;
  HG_GUARD_END
}

int hg_comm_init(hg_engine* e, const uint8_t* id, int rank, int world) {
  HG_GUARD_BEGIN
  if (!e || !id || world < 1 || rank < 0 || rank >= world) return set_error(HG_ERR_INVALID, "bad argument");
  NcclApi* api = nccl_api();
  if (!api->err.empty()) return set_error(HG_ERR_UNSUPPORTED, api->err);
  std::lock_guard<std::mutex> g(e->mu);
  if (e->comm) return set_error(HG_ERR_INVALID, "communicator already initialised");
  CU_TRY(cudaSetDevice(e->device));
  auto c = std::make_unique<hg_comm>();
  c->rank = rank;
  c->world = world;
  nccl_uid u;
  std::memcpy(u.internal, id, HG_COMM_ID_BYTES);
  NCCL_TRY(api, api->CommInitRank(&c->comm, world, u, rank));
  CU_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  CU_TRY(cudaEventCreateWithFlags(&c->ev_packed, cudaEventDisableTiming));
  CU_TRY(cudaEventCreateWithFlags(&c->ev_done, cudaEventDisableTiming));
  CU_TRY(cudaMalloc(&c->d_sizes, (size_t(world) + 1) * 8));
  CU_TRY(cudaMalloc(&c->d_n, 64));
  CU_TRY(cudaMallocHost(&c->h_sizes, (size_t(world) + 1) * 8));
  e->comm = c.release();
  return HG_OK;
  HG_GUARD_END
}

int hg_comm_destroy(hg_engine* e) {
  HG_GUARD_BEGIN
  if (!e) return set_error(HG_ERR_INVALID, "null engine");
  std::lock_guard<std::mutex> g(e->mu);
  cudaSetDevice(e->device);
  hg_comm_free(e->comm);
  e->comm = nullptr;
  return HG_OK;
  HG_GUARD_END
}

int hg_comm_sync(hg_engine* e) {
  HG_GUARD_BEGIN
  if (!e || !e->comm) return set_error(HG_ERR_INVALID, "no communicator");
  CU_TRY(cudaSetDevice(e->device));
  CU_TRY(cudaStreamSynchronize(e->comm->stream));
  return HG_OK;
  HG_GUARD_END
}

int hg_agg_combine(hg_engine* e, uint32_t mode, uint64_t capacity_hint, hg_agg_combined* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  if (mode > HG_COMBINE_REDUCE) return set_error(HG_ERR_INVALID, "combine mode");
  std::lock_guard<std::mutex> g(e->mu);
  hg_comm* c = e->comm;
  if (!c) return set_error(HG_ERR_INVALID, "hg_comm_init has not been called on this engine");
  NcclApi* api = nccl_api();
  CU_TRY(cudaSetDevice(e->device));
  const uint64_t G = e->last_agg.num_groups;
  std::memset(out, 0, sizeof(*out));
  uint64_t cap = capacity_hint;
  if (cap == 0) {
    // agree on the block width: all-gather of the group counts (one small collective + one host sync)
    CU_TRY(cudaStreamSynchronize(c->stream));
    c->h_sizes[c->world] = G;
    CU_TRY(cudaMemcpyAsync(c->d_sizes + c->world, c->h_sizes + c->world, 8, cudaMemcpyHostToDevice, c->stream));
    NCCL_TRY(api, api->AllGather(c->d_sizes + c->world, c->d_sizes, 1, kNcclInt64, c->comm, c->stream));
    CU_TRY(cudaMemcpyAsync(c->h_sizes, c->d_sizes, size_t(c->world) * 8, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    for (int r = 0; r < c->world; r++) cap = std::max<uint64_t>(cap, c->h_sizes[r]);
    if (cap == 0) cap = 1;
  } else if (G > cap) return set_error(HG_ERR_INVALID, "partial aggregate larger than the agreed capacity");
  if (uint64_t(c->world) * cap >= 0xfffffff0ull) return set_error(HG_ERR_UNSUPPORTED, "combined table larger than 2^32 rows");
  // the previous combine may still be reading the buffers
  CU_TRY(cudaStreamSynchronize(c->stream));
  int rc = ensure_buffers(c, cap, mode == HG_COMBINE_REDUCE);
  if (rc) return rc;
  cap = c->cap;                              // blocks keep the allocated width (stable addresses, no re-agreement)
  // pack behind the scan on the engine stream, hand over to the combine stream
  AggOut in{const_cast<void*>(e->last_agg.d_gkey), const_cast<int64_t*>(e->last_agg.d_bucket), const_cast<uint64_t*>(e->last_agg.d_count),
            const_cast<double*>(e->last_agg.d_sum), const_cast<double*>(e->last_agg.d_min), const_cast<double*>(e->last_agg.d_max)};
  Launch L = e->L();
  k::pack_agg(L, in, e->last_gwidth, G, cap, c->d_send);
  CU_TRY(cudaEventRecord(c->ev_packed, e->stream));
  CU_TRY(cudaStreamWaitEvent(c->stream, c->ev_packed, 0));
  NCCL_TRY(api, api->AllGather(c->d_send, c->d_recv, size_t(6) * cap, kNcclInt64, c->comm, c->stream));
  out->capacity = cap;
  out->world = uint32_t(c->world);
  out->d_blocks = reinterpret_cast<const int64_t*>(c->d_recv);
  if (mode == HG_COMBINE_REDUCE) {
    Launch LC{c->stream, &c->launches};
    const uint32_t total = uint32_t(uint64_t(c->world) * cap);
    red_collect_kernel<<<1, 256, 0, c->stream>>>(c->d_recv, uint32_t(c->world), cap, c->d_v1, c->d_n);
    // stable sort by bucket, then by the typed group key (LSD over the composite)
    red_keys_kernel<<<kNumSMs, 256, 0, c->stream>>>(c->d_recv, cap, c->d_v1, c->d_n, 0, e->last_gtype, c->d_k1);
    uint32_t* v = c->d_v1;
    uint32_t* vt = c->d_v2;
    if (k::radix_sort_pairs(LC, c->d_k1, v, c->d_k2, vt, c->d_n, total, 64, c->d_counts)) std::swap(v, vt);
    red_keys_kernel<<<kNumSMs, 256, 0, c->stream>>>(c->d_recv, cap, v, c->d_n, 1, e->last_gtype, c->d_k1);
    if (k::radix_sort_pairs(LC, c->d_k1, v, c->d_k2, vt, c->d_n, total, 64, c->d_counts)) std::swap(v, vt);
    red_heads_kernel<<<kNumSMs, 256, 0, c->stream>>>(c->d_recv, cap, v, c->d_n, total, c->d_head);
    k::compact_flags(LC, c->d_head, total, c->d_tmp, c->d_seg, c->d_n + 1);
    red_reduce_kernel<<<kNumSMs, 256, 0, c->stream>>>(c->d_recv, cap, v, c->d_n, c->d_seg, c->d_n + 1, c->red_cap, c->d_out);
    CU_TRY(cudaGetLastError());
    uint32_t hg = 0;
    CU_TRY(cudaMemcpyAsync(&hg, c->d_n + 1, 4, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(cudaStreamSynchronize(c->stream));
    out->num_groups = hg;
    out->reduced_capacity = c->red_cap;
    out->d_reduced = reinterpret_cast<const int64_t*>(c->d_out);
  }
  CU_TRY(cudaEventRecord(c->ev_done, c->stream));
  return HG_OK;
  HG_GUARD_END
}

}  // extern "C"
