// bloom.h — Parquet split-block bloom filters (SBBF, parquet-format BloomFilter.md), shared by the writer's bloom_build_kernel
// (sst_writer.cu), the device probes of the scan planner (engine.cu, fused_scan.cu) and the host probe (engine.cu, inspect.cpp).
//
// A filter is numBytes / 32 blocks of eight 32-bit words.  A value's hash h is xxHash64 (seed 0) of its PLAIN physical bytes
// (4 for INT32 / FLOAT, 8 for INT64 / DOUBLE); the upper half of h picks the block, the lower half sets one bit in each word.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define BLOOM_FN __host__ __device__ __forceinline__
#else
#define BLOOM_FN inline
#endif

namespace horae {
namespace bloom {

constexpr uint32_t kMinBytes = 32, kMaxBytes = 128u << 20;   // the spec's bounds on numBytes
constexpr uint32_t kDefaultBytes = 1u << 20;                 // parquet-rs / pyarrow defaults: ndv 1,000,000, fpp 0.05

constexpr uint64_t kP1 = 0x9E3779B185EBCA87ull, kP2 = 0xC2B2AE3D27D4EB4Full, kP3 = 0x165667B19E3779F9ull, kP4 = 0x85EBCA77C2B2AE63ull,
                   kP5 = 0x27D4EB2F165667C5ull;

BLOOM_FN uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
BLOOM_FN uint64_t avalanche(uint64_t h) {
  h ^= h >> 33; h *= kP2;
  h ^= h >> 29; h *= kP3;
  h ^= h >> 32;
  return h;
}
// xxHash64, seed 0, of the 4 little-endian bytes of v
BLOOM_FN uint64_t xxh64_4(uint32_t v) {
  uint64_t h = kP5 + 4;
  h ^= uint64_t(v) * kP1;
  h = rotl64(h, 23) * kP2 + kP3;
  return avalanche(h);
}
// xxHash64, seed 0, of the 8 little-endian bytes of v
BLOOM_FN uint64_t xxh64_8(uint64_t v) {
  uint64_t h = kP5 + 8;
  h ^= rotl64(v * kP2, 31) * kP1;
  h = rotl64(h, 27) * kP1 + kP4;
  return avalanche(h);
}

BLOOM_FN uint32_t block_of(uint64_t h, uint32_t num_blocks) { return uint32_t(((h >> 32) * uint64_t(num_blocks)) >> 32); }
// mask word i (0..7) of the block: one bit chosen by the salted lower half of the hash
BLOOM_FN uint32_t mask_word(uint64_t h, int i) {
  const uint32_t salt = i == 0 ? 0x47b6137bu : i == 1 ? 0x44974d91u : i == 2 ? 0x8824ad5bu : i == 3 ? 0xa2b7289du
                      : i == 4 ? 0x705495c7u : i == 5 ? 0x2df1424bu : i == 6 ? 0x9efc4947u : 0x5c6bfb31u;
  return 1u << ((uint32_t(h) * salt) >> 27);
}
// the filter whose bitset starts at `bits` (num_blocks * 32 bytes, little-endian words, any alignment) may hold the value hashed to h
BLOOM_FN bool may_contain(const uint8_t* bits, uint32_t num_blocks, uint64_t h) {
  const uint8_t* b = bits + uint64_t(block_of(h, num_blocks)) * 32;
  for (int i = 0; i < 8; i++) {
    const uint32_t w = uint32_t(b[4 * i]) | (uint32_t(b[4 * i + 1]) << 8) | (uint32_t(b[4 * i + 2]) << 16) | (uint32_t(b[4 * i + 3]) << 24);
    if (!(w & mask_word(h, i))) return false;
  }
  return true;
}

}  // namespace bloom
}  // namespace horae
