// sst_writer.h — GPU Parquet page encoder + SST assembly (sst_writer.cu).
#pragma once
#include <vector>

#include "engine_internal.h"

namespace horae {
namespace writer {
// The writer options of a call, checked and with their defaults applied
struct WriteOpts {
  std::vector<hg_column_write_opts> cols;   // one per schema column
  uint32_t max_row_group_size;              // 0 in hg_write_props -> 8192
  uint32_t bloom_filter_bytes;              // 0 in hg_write_props -> bloom::kDefaultBytes
  bool sorting_columns;
};
// The writer options of every column (props->columns, or PLAIN with props->compression when it is NULL), checked: HG_ERR_UNSUPPORTED
// naming the column for a Binary column, an unknown codec, an encoding other than PLAIN / DELTA_BINARY_PACKED, or DELTA on a float column.
int resolve_write_opts(const hg_schema_desc* schema, const hg_write_props* props, WriteOpts* out);
struct ColIn {
  const void* vals;         // dense device column, native width
  const uint8_t* valid;     // one byte per row (1 = non-null) or nullptr
  uint32_t type, width;
};
// A cudaMallocHost'ed SST image, freed when its owner goes out of scope
struct PinnedImage {
  uint8_t* p = nullptr;
  uint64_t size = 0;
  PinnedImage() = default;
  PinnedImage(const PinnedImage&) = delete;
  PinnedImage& operator=(const PinnedImage&) = delete;
  ~PinnedImage() { if (p) cudaFreeHost(p); }
};
// Encodes R rows of the schema's device columns as one SST (Parquet) image.  Runs on the engine's stream; synchronises.
int write_sst(hg_engine* e, const hg_schema_desc* schema, const ColIn* cols, uint32_t R, const WriteOpts& wo, PinnedImage* out);
}  // namespace writer
}  // namespace horae
