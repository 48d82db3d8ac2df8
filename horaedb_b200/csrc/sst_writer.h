// sst_writer.h — GPU Parquet page encoder + SST assembly (sst_writer.cu).
#pragma once
#include <vector>

#include "engine_internal.h"

namespace horae {
namespace writer {
// The writer options of every column (props->columns, or PLAIN with props->compression when it is NULL), checked: HG_ERR_UNSUPPORTED
// naming the column for a Binary column, an unknown codec, an encoding other than PLAIN / DELTA_BINARY_PACKED, or DELTA on a float column.
int resolve_write_opts(const hg_schema_desc* schema, const hg_write_props* props, std::vector<hg_column_write_opts>* out);
struct ColIn {
  const void* vals;         // dense device column, native width
  const uint8_t* valid;     // one byte per row (1 = non-null) or nullptr
  uint32_t type, width;
};
// Encodes R rows of `ncols` device columns as one SST (Parquet) image.  *host_out = cudaMallocHost'ed buffer of *size_out
// bytes (the caller frees it with cudaFreeHost).  Runs on the engine's stream; synchronises.
int write_sst(hg_engine* e, const hg_schema_desc* schema, const ColIn* cols, uint32_t ncols, uint32_t R, const hg_write_props* props,
              uint8_t** host_out, uint64_t* size_out);
}  // namespace writer
}  // namespace horae
