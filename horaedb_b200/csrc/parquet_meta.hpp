// parquet_meta.hpp — host-side Parquet footer + page-header walk for the SST format the reference writes
// (build_write_props, storage.rs:258-298; WriteConfig::default, config.rs:120-133).
//
// In the reference this work happens inside parquet-rs (ParquetExec / DefaultParquetFileReaderFactory,
// read.rs:66-93, 456-465).  Here the host only produces a flat page table; every byte of page payload is decoded on
// the GPU (kernels.cu).  Thrift compact protocol and the FileMetaData / PageHeader field ids follow the Apache
// Parquet format specification (parquet.thrift).
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "device_types.h"   // PhysType, Codec, Encoding, PageType

namespace horae {

struct ColumnStats {
  bool has_min = false, has_max = false, has_null_count = false;
  uint8_t min[8] = {0}, max[8] = {0};   // min_value / max_value of 1 to 8 bytes (has_min / has_max), zero padded
  int64_t null_count = 0;
  // BYTE_ARRAY chunks: the whole min_value / max_value (any length, empty included) at [off, off + len) of FileMetaData::stat_bytes.
  // The deprecated min / max fields are never read: old writers ordered them as signed bytes.
  bool has_bin_min = false, has_bin_max = false;
  uint32_t bin_min_off = 0, bin_min_len = 0, bin_max_off = 0, bin_max_len = 0;
};

struct PageMeta {
  uint64_t payload_off = 0;  // file offset of the first byte after the page header
  uint32_t comp_size = 0, uncomp_size = 0, num_values = 0;
  uint32_t v2_def_len = 0, v2_rep_len = 0;
  uint8_t page_type = 0, encoding = 0, v2_compressed = 1;
  uint8_t def_level_encoding = 3;   // V1 pages: RLE (3), or the deprecated BIT_PACKED (4), which has no length in front of the levels
};

struct ChunkMeta {
  int phys_type = 0, codec = 0;
  int64_t num_values = 0, data_page_offset = 0, dict_page_offset = -1, total_compressed = 0;
  ColumnStats stats;
  uint32_t first_page = 0, num_pages = 0;   // into FileMetaData::pages (data pages only)
  uint64_t scratch_bytes = 0;               // bytes of decode scratch this chunk needs (chunk_scratch.h)
  bool has_dict_page = false;
  uint64_t dict_payload_off = 0;            // dictionary page (RLE_DICTIONARY chunks): PLAIN values
  uint32_t dict_comp_size = 0, dict_uncomp_size = 0, dict_num_values = 0;
  int64_t bloom_offset = -1;                // ColumnMetaData.bloom_filter_offset (BloomFilterHeader), -1: absent
  int32_t bloom_length = -1;                // ColumnMetaData.bloom_filter_length (header + bitset), when has_bloom_length
  bool has_bloom_length = false;
};

struct RowGroupMeta {
  int64_t num_rows = 0, first_row = 0;
  std::vector<ChunkMeta> cols;
};

struct FileMetaData {
  int ncols = 0;
  std::vector<int> repetition;  // per leaf: 0 required, 1 optional
  std::vector<int> phys_types;
  std::vector<std::string> names;
  int64_t num_rows = 0;
  std::vector<RowGroupMeta> rgs;
  std::vector<PageMeta> pages;
  std::vector<uint8_t> stat_bytes;   // the BYTE_ARRAY chunks' statistics bytes (ColumnStats::bin_*)
};

// Parses the footer and walks every column chunk's page headers.  Returns false and fills *err on malformed input.
bool parse_parquet(const uint8_t* data, size_t len, FileMetaData* out, std::string* err);

// The chunk's split-block bloom filter, if it is one this reader can probe: a BloomFilterHeader with numBytes a power of two in
// [32 B, 128 MiB], algorithm BLOCK, hash XXHASH, compression UNCOMPRESSED, and header + bitset inside bloom_filter_length (when given)
// and inside the file.  Anything else (absent, damaged, unknown) returns false: the filter is ignored.
bool bloom_bitset(const uint8_t* data, size_t len, const ChunkMeta& cm, uint64_t* bitset_off, uint32_t* num_bytes);

}  // namespace horae
