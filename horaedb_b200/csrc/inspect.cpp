// inspect.cpp — host-only SST inspection entry points (hg_parquet_inspect, hg_parquet_chunk_info, hg_parquet_bloom_*): the footer / page-header
// facts the planner works from, exposed so that the CPU test-suite can check parquet_meta.cpp against pyarrow without a GPU.
#include <string>

#include "../../include/horae_gpu.h"
#include "bloom.h"
#include "parquet_meta.hpp"

#include <new>
int set_error(int code, const std::string& msg);   // engine.cu
#define HG_GUARD_BEGIN try {
#define HG_GUARD_END                                                                                              \
  }                                                                                                               \
  catch (const std::bad_alloc&) { return set_error(HG_ERR_OOM, "host allocation failed"); }                      \
  catch (const std::exception& ex) { return set_error(HG_ERR_INTERNAL, std::string("exception: ") + ex.what()); } \
  catch (...) { return set_error(HG_ERR_INTERNAL, "unknown exception"); }

int set_error(int code, const std::string& msg);   // engine.cu (thread-local message behind hg_last_error)

using namespace horae;

extern "C" {

int hg_parquet_inspect(const uint8_t* data, uint64_t size, hg_parquet_summary* out) {
  HG_GUARD_BEGIN
  if (!data || !out) return set_error(HG_ERR_INVALID, "null argument");
  FileMetaData m;
  std::string err;
  if (!parse_parquet(data, size_t(size), &m, &err)) return set_error(HG_ERR_FORMAT, err);
  hg_parquet_summary s{};
  s.num_rows = uint64_t(m.num_rows);
  s.num_row_groups = uint32_t(m.rgs.size());
  s.num_columns = uint32_t(m.ncols);
  s.num_data_pages = m.pages.size();
  for (const PageMeta& p : m.pages) {
    s.sum_page_values += p.num_values;
    s.sum_uncompressed_bytes += p.uncomp_size;
    s.sum_compressed_bytes += p.comp_size;
  }
  for (const RowGroupMeta& rg : m.rgs)
    for (const ChunkMeta& c : rg.cols) {
      if (c.codec >= 0 && c.codec < 32) s.codec_mask |= 1u << c.codec;
      if (c.num_pages > s.max_pages_per_chunk) s.max_pages_per_chunk = c.num_pages;
    }
  *out = s;
  return HG_OK;
  HG_GUARD_END
}

int hg_parquet_chunk_info(const uint8_t* data, uint64_t size, uint32_t row_group, uint32_t column, hg_parquet_chunk* out) {
  HG_GUARD_BEGIN
  if (!data || !out) return set_error(HG_ERR_INVALID, "null argument");
  FileMetaData m;
  std::string err;
  if (!parse_parquet(data, size_t(size), &m, &err)) return set_error(HG_ERR_FORMAT, err);
  if (row_group >= m.rgs.size() || column >= uint32_t(m.ncols)) return set_error(HG_ERR_INVALID, "row group / column out of range");
  const RowGroupMeta& rg = m.rgs[row_group];
  const ChunkMeta& c = rg.cols[column];
  hg_parquet_chunk o{};
  o.num_rows = uint64_t(rg.num_rows);
  o.num_values = uint64_t(c.num_values);
  o.data_page_offset = c.data_page_offset;
  o.total_compressed_size = c.total_compressed;
  o.null_count = c.stats.has_null_count ? c.stats.null_count : -1;
  o.has_min_max = c.stats.has_min && c.stats.has_max;
  for (int i = 0; i < 8; i++) { o.min[i] = c.stats.min[i]; o.max[i] = c.stats.max[i]; }
  o.physical_type = uint32_t(c.phys_type);
  o.codec = uint32_t(c.codec);
  o.num_pages = c.num_pages;
  if (c.num_pages) {
    const PageMeta& p = m.pages[c.first_page];
    o.first_page_payload_offset = p.payload_off;
    o.first_page_num_values = p.num_values;
    o.first_page_type = p.page_type;
  }
  *out = o;
  return HG_OK;
  HG_GUARD_END
}

int hg_parquet_bloom_info(const uint8_t* data, uint64_t size, uint32_t row_group, uint32_t column, hg_parquet_bloom* out) {
  HG_GUARD_BEGIN
  if (!data || !out) return set_error(HG_ERR_INVALID, "null argument");
  FileMetaData m;
  std::string err;
  if (!parse_parquet(data, size_t(size), &m, &err)) return set_error(HG_ERR_FORMAT, err);
  if (row_group >= m.rgs.size() || column >= uint32_t(m.ncols)) return set_error(HG_ERR_INVALID, "row group / column out of range");
  const ChunkMeta& c = m.rgs[row_group].cols[column];
  hg_parquet_bloom o{};
  o.offset = c.bloom_offset;
  o.length = c.bloom_length;
  o.usable = bloom_bitset(data, size_t(size), c, &o.bitset_offset, &o.num_bytes) ? 1 : 0;
  if (!o.usable) { o.bitset_offset = 0; o.num_bytes = 0; }
  *out = o;
  return HG_OK;
  HG_GUARD_END
}

int hg_parquet_bloom_probe(const uint8_t* data, uint64_t size, uint32_t row_group, uint32_t column, const void* value, uint32_t len,
                           int* maybe) {
  HG_GUARD_BEGIN
  if (!value || !maybe) return set_error(HG_ERR_INVALID, "null argument");
  if (len != 4 && len != 8) return set_error(HG_ERR_INVALID, "bloom probe: a PLAIN value is 4 or 8 bytes");
  hg_parquet_bloom b;
  const int rc = hg_parquet_bloom_info(data, size, row_group, column, &b);
  if (rc) return rc;
  *maybe = 1;
  if (!b.usable) return HG_OK;
  uint64_t v = 0;
  std::memcpy(&v, value, len);
  const uint64_t h = len == 8 ? bloom::xxh64_8(v) : bloom::xxh64_4(uint32_t(v));
  *maybe = bloom::may_contain(data + b.bitset_offset, b.num_bytes / 32, h) ? 1 : 0;
  return HG_OK;
  HG_GUARD_END
}

}  // extern "C"
