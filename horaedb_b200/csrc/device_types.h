// device_types.h — plain structs shared by the host engine and the CUDA kernels (HBM-resident page tables and
// per-scan descriptors).  Names follow the reference's domain: SSTs, row groups, column chunks, pages.
#pragma once
#include <cstdint>

namespace horae {

enum : uint32_t { T_U8 = 0, T_I8, T_U16, T_I16, T_U32, T_I32, T_U64, T_I64, T_F32, T_F64, T_BINARY };
enum : uint32_t { OP_EQ = 0, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_IN };

// Parquet's numbers for these (parquet.thrift), as the footer and the page headers carry them
enum PhysType : int { PT_BOOLEAN = 0, PT_INT32 = 1, PT_INT64 = 2, PT_INT96 = 3, PT_FLOAT = 4, PT_DOUBLE = 5, PT_BYTE_ARRAY = 6, PT_FLBA = 7 };
enum Codec : int { CODEC_UNCOMPRESSED = 0, CODEC_SNAPPY = 1, CODEC_ZSTD = 6 };
enum Encoding : int { ENC_PLAIN = 0, ENC_PLAIN_DICT = 2, ENC_RLE = 3, ENC_DELTA_BINARY_PACKED = 5, ENC_DELTA_LENGTH_BYTE_ARRAY = 6, ENC_DELTA_BYTE_ARRAY = 7, ENC_RLE_DICT = 8 };
enum PageType : int { PAGE_DATA = 0, PAGE_INDEX = 1, PAGE_DICT = 2, PAGE_DATA_V2 = 3 };

#if defined(__CUDACC__)
#define HORAE_HD __host__ __device__ __forceinline__
#else
#define HORAE_HD inline
#endif
// Floats compare in IEEE-754 totalOrder, like arrow-rs 53's comparison kernels behind DataFusion's FilterExec and
// PruningPredicate (read.rs:459-470): -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN.  The key maps f64 bits to an
// unsigned integer with the same order.
HORAE_HD uint64_t f64_total_order_key(uint64_t bits) { return bits ^ ((bits >> 63) ? ~0ull : (1ull << 63)); }
HORAE_HD int cmp_f64_total(uint64_t a, uint64_t b) {
  const uint64_t x = f64_total_order_key(a), y = f64_total_order_key(b);
  return x < y ? -1 : (x > y ? 1 : 0);
}

// One data page (resident next to its SST's bytes).  32 bytes.
struct PageDev {
  uint64_t payload_off;   // byte offset of the page payload in the file
  uint32_t comp_size, uncomp_size, num_values;
  uint32_t v2_def_len, v2_rep_len;
  uint8_t page_type;      // PAGE_DATA (V1) or PAGE_DATA_V2
  uint8_t encoding, v2_compressed, _pad;
};

// One column chunk, indexed [row_group * ncols + column].  32 bytes.
struct ChunkDev {
  uint32_t first_page, num_pages;
  uint32_t scratch_bytes;  // decode scratch needed by this chunk (layout: chunk_scratch.h)
  uint8_t phys;            // PhysType
  uint8_t codec;           // CODEC_UNCOMPRESSED, CODEC_SNAPPY or CODEC_ZSTD
  uint8_t optional;        // max definition level 1
  uint8_t stored;          // Snappy, one V1 page, stream = 1-2 literals whose value bytes are row-aligned: readable in place
  // dictionary page of the chunk (RLE_DICTIONARY data pages index into its PLAIN values); dict_uncomp == 0: none
  uint64_t dict_payload_off;
  uint32_t dict_comp, dict_uncomp;
};

// One DELTA_BYTE_ARRAY page of a scan call.  decode_chunks sizes it (everything but out_off); the host scans `bytes` into out_off,
// and dba_materialise writes the page's values at out_off of the call's value buffer.
struct DbaPage {
  const uint32_t* lens;    // prefix lengths [nv], then suffix lengths [nv] (the page's image in scratch), of the non-null values
  const uint8_t* suffix;   // the suffix bytes, back to back
  uint64_t bytes;          // materialised bytes of the page's values
  uint64_t out_off;        // first byte of the page's values in the call's value buffer
  uint32_t n;              // non-null values (0 when the page failed validation)
  uint32_t nv;             // rows of the page
  uint32_t row;            // first row of the page in the decoded columns
  uint32_t ci;             // ColSel index of the column
};

struct SstDev {
  const uint8_t* bytes;
  const PageDev* pages;
  const ChunkDev* chunks;
  uint32_t ncols, nrgs;
};

// A row group selected by the planner (after statistics pruning).
struct RgSel {
  uint32_t sst, rg;        // index into the scan's SstDev table / row group in that SST
  uint32_t out_row;        // first row of this row group in the decoded columns
  uint32_t num_rows;
  uint64_t scratch_off;    // base of this row group's decompression scratch
};

// A column to decode.
struct ColSel {
  uint32_t col, type, out_width, _pad;
  void* out_vals;          // Binary columns: one `const uint8_t*` per row pointing at the value's bytes (page payload / scratch)
  uint8_t* out_valid;      // one byte per row (1 = non-null)
  uint32_t* out_lens;      // Binary columns only: byte length per row
};

// A decoded column.
struct ColView {
  const void* vals;
  const uint8_t* valid;
  uint32_t type, width;
  const uint32_t* lens;    // Binary columns only (vals = per-row byte pointers), else nullptr
};

struct PredDev {
  ColView col;
  uint32_t op, n_in;       // n_in: OP_IN list length
  uint64_t lit;            // literal bit pattern in the column's widened domain (i64 / u64 / f64)
  const uint64_t* in_list; // OP_IN: device array of n_in literals
};

constexpr int MAX_PREDS = 8;
constexpr int MAX_PK = 4;
constexpr int MAX_COLS = 32;

struct PredSet { PredDev p[MAX_PREDS]; int n; };
struct PkSet { ColView c[MAX_PK]; int n; };

// 32-byte sort record of the k-way merge: (normalised PK : 128 bit, __seq__, row id) compared lexicographically.
struct alignas(16) SortRec { uint64_t k0, k1, seq, row; };

struct AggSpecDev {
  ColView group, ts, value;
  int has_group, has_ts, has_value;
  int64_t window_ms;
};

struct AggOut {
  void* gkey;            // native width of the group column
  int64_t* bucket;
  uint64_t* count;
  double* sum;
  double* min;
  double* max;
};

}  // namespace horae
