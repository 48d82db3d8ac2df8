// device_types.h — plain structs shared by the host engine and the CUDA kernels (HBM-resident page tables and
// per-scan descriptors).  Names follow the reference's domain: SSTs, row groups, column chunks, pages.
#pragma once
#include <cstdint>
#include <cstring>

namespace horae {

enum : uint32_t { T_U8 = 0, T_I8, T_U16, T_I16, T_U32, T_I32, T_U64, T_I64, T_F32, T_F64, T_BINARY };
enum : uint32_t { OP_EQ = 0, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_IN, OP_IN_SET };

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

// ---- The comparison domain.  Predicates, statistics, merge / GROUP BY keys and the NCCL combine all compare values widened
// to 64 bits (signed -> i64 bits, unsigned -> u64, floats -> f64 bits); order_key maps a widened value to an unsigned key
// with the same order.  This is the one definition of both rules.
HORAE_HD uint32_t type_width(uint32_t t) {
  switch (t) {
    case T_U8: case T_I8: return 1;
    case T_U16: case T_I16: return 2;
    case T_U32: case T_I32: case T_F32: return 4;
    default: return 8;
  }
}
HORAE_HD bool type_is_signed(uint32_t t) { return t == T_I8 || t == T_I16 || t == T_I32 || t == T_I64; }
HORAE_HD bool type_is_float(uint32_t t) { return t == T_F32 || t == T_F64; }

// native-width bits of a value (zero-extended) -> the comparison domain
HORAE_HD uint64_t widen(uint64_t raw, uint32_t t) {
  switch (t) {
    case T_I8: return uint64_t(int64_t(int8_t(raw)));
    case T_I16: return uint64_t(int64_t(int16_t(raw)));
    case T_I32: return uint64_t(int64_t(int32_t(raw)));
    case T_F32: {
#if defined(__CUDA_ARCH__)
      return uint64_t(__double_as_longlong(double(__uint_as_float(uint32_t(raw)))));
#else
      const uint32_t b = uint32_t(raw);
      float f;
      std::memcpy(&f, &b, 4);
      const double d = f;
      uint64_t v;
      std::memcpy(&v, &d, 8);
      return v;
#endif
    }
    default: return raw;
  }
}
HORAE_HD uint64_t order_flip(uint32_t t) { return type_is_signed(t) ? (1ull << 63) : 0ull; }
HORAE_HD uint64_t order_key(uint64_t widened, uint32_t t) {
  if (type_is_float(t)) return f64_total_order_key(widened);
  return type_is_signed(t) ? widened ^ (1ull << 63) : widened;
}
// a widened float that is a NaN (any sign or payload)
HORAE_HD bool widened_is_nan(uint64_t widened, uint32_t t) {
  return type_is_float(t) && (widened & ~(1ull << 63)) > 0x7ff0000000000000ull;
}
// The inverse of order_key(widen(x)): an order key -> the PLAIN physical bits of its value (1-, 2- and 4-byte integers as INT32, f32 as
// FLOAT; the f64 -> f32 step is exact for a value widened from a float)
HORAE_HD uint64_t order_key_to_plain(uint64_t key, uint32_t t) {
  const uint64_t w = type_is_float(t) ? key ^ ((key >> 63) ? (1ull << 63) : ~0ull) : key ^ order_flip(t);
  switch (t) {
    case T_I8: case T_I16: case T_I32: return uint32_t(w);
    case T_F32: {
#if defined(__CUDA_ARCH__)
      return __float_as_uint(float(__longlong_as_double((long long)w)));
#else
      double d;
      std::memcpy(&d, &w, 8);
      const float f = float(d);
      uint32_t b;
      std::memcpy(&b, &f, 4);
      return b;
#endif
    }
    default: return w;
  }
}

// Three-way compare of two widened values by comparison class (the fused kernel keeps the class per column)
enum : uint32_t { C_UNSIGNED = 0, C_SIGNED = 1, C_FLOAT = 2 };
HORAE_HD uint32_t cmp_class(uint32_t t) { return type_is_float(t) ? C_FLOAT : (type_is_signed(t) ? C_SIGNED : C_UNSIGNED); }
HORAE_HD int cmp_widened(uint64_t a, uint64_t b, uint32_t cls) {
  if (cls == C_FLOAT) return cmp_f64_total(a, b);
  if (cls == C_SIGNED) {
    const int64_t x = int64_t(a), y = int64_t(b);
    return x < y ? -1 : (x > y ? 1 : 0);
  }
  return a < b ? -1 : (a > b ? 1 : 0);
}
// `value op literal` from c = cmp_widened(value, literal) (OP_IN is the caller's loop of OP_EQ)
HORAE_HD bool op_holds(int c, uint32_t op) {
  switch (op) {
    case OP_EQ: return c == 0;
    case OP_NE: return c != 0;
    case OP_LT: return c < 0;
    case OP_LE: return c <= 0;
    case OP_GT: return c > 0;
    default: return c >= 0;
  }
}
// DataFusion PruningPredicate's min/max rewrite (read.rs:613) of `col op lit`: false when no value in [mn, mx] can pass
HORAE_HD bool minmax_may_match(uint64_t mn, uint64_t mx, uint64_t lit, uint32_t op, uint32_t cls) {
  switch (op) {
    case OP_EQ: return cmp_widened(mn, lit, cls) <= 0 && cmp_widened(lit, mx, cls) <= 0;
    case OP_NE: return cmp_widened(mn, lit, cls) != 0 || cmp_widened(lit, mx, cls) != 0;
    case OP_LT: return cmp_widened(mn, lit, cls) < 0;
    case OP_LE: return cmp_widened(mn, lit, cls) <= 0;
    case OP_GT: return cmp_widened(mx, lit, cls) > 0;
    default: return cmp_widened(mx, lit, cls) >= 0;
  }
}
// `col IN (set)` for large sets (OP_IN_SET).  The set is held as the order_key of every member, sorted and unique.  The slice [*lo, *hi)
// of the set whose keys lie in [kmin, kmax], by two binary searches; true when it holds a key.  With kmin / kmax the keys of a chunk's
// statistics this is the min/max rewrite of the predicate (some member inside [min, max]); with the bounds of a tile of rows it is the
// part of the set those rows can match.
HORAE_HD bool key_set_slice(const uint64_t* keys, uint32_t n, uint64_t kmin, uint64_t kmax, uint32_t* lo, uint32_t* hi) {
  uint32_t a = 0, b = n;
  while (a < b) { const uint32_t m = a + ((b - a) >> 1); if (keys[m] < kmin) a = m + 1; else b = m; }
  *lo = a;
  b = n;
  while (a < b) { const uint32_t m = a + ((b - a) >> 1); if (keys[m] <= kmax) a = m + 1; else b = m; }
  *hi = a;
  return *lo < *hi;
}

// ---- Binary values (Arrow Binary / Parquet BYTE_ARRAY) order as arrow-rs BinaryArray does: unsigned bytes lexicographically, a proper
// prefix first.  A value's KEY is its first 8 bytes big-endian, zero padded: keys order like the values whenever they differ, so most
// compares are one u64 compare; equal keys fall through to the bytes from offset 8 and the lengths.  No access leaves [p, p + len).
HORAE_HD uint64_t bytes_load_be64(const uint8_t* p) {   // 8 bytes at any alignment, big-endian
#if defined(__CUDA_ARCH__)
  // the aligned words holding p[0] and p[7]: never a byte outside them, so never across a page
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint64_t* w = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
  const uint32_t sh = uint32_t(a & 7) * 8;
  const uint64_t le = sh ? (w[0] >> sh) | (w[1] << (64 - sh)) : w[0];
  const uint32_t lo = uint32_t(le), hi = uint32_t(le >> 32);
  return (uint64_t(__byte_perm(lo, 0, 0x0123)) << 32) | __byte_perm(hi, 0, 0x0123);
#else
  uint64_t le;
  std::memcpy(&le, p, 8);
  return __builtin_bswap64(le);
#endif
}
HORAE_HD uint64_t bytes_key(const uint8_t* p, uint64_t len) {
  if (len >= 8) return bytes_load_be64(p);
  uint64_t k = 0;
  for (uint32_t i = 0; i < uint32_t(len); i++) k |= uint64_t(p[i]) << (56 - 8 * i);
  return k;
}
// three-way compare of a and b given their keys
HORAE_HD int cmp_bytes_keyed(uint64_t ka, const uint8_t* a, uint64_t la, uint64_t kb, const uint8_t* b, uint64_t lb) {
  if (ka != kb) return ka < kb ? -1 : 1;
  const uint64_t n = la < lb ? la : lb;
  for (uint64_t i = 8; i < n; i += 8) {
    const uint64_t x = bytes_key(a + i, n - i), y = bytes_key(b + i, n - i);
    if (x != y) return x < y ? -1 : 1;
  }
  return la < lb ? -1 : (la > lb ? 1 : 0);
}
HORAE_HD int cmp_bytes(const uint8_t* a, uint64_t la, const uint8_t* b, uint64_t lb) {
  return cmp_bytes_keyed(bytes_key(a, la), a, la, bytes_key(b, lb), b, lb);
}
// The min/max rewrite for Binary chunks.  Their min_value / max_value are BOUNDS (a writer may truncate them: min_value <= every value
// <= max_value), so `<>` never prunes; otherwise the rule of minmax_may_match.
HORAE_HD bool bytes_minmax_may_match(const uint8_t* mn, uint64_t lmn, const uint8_t* mx, uint64_t lmx, const uint8_t* lit, uint64_t llit,
                                     uint32_t op) {
  switch (op) {
    case OP_EQ: return cmp_bytes(mn, lmn, lit, llit) <= 0 && cmp_bytes(lit, llit, mx, lmx) <= 0;
    case OP_NE: return true;
    case OP_LT: return cmp_bytes(mn, lmn, lit, llit) < 0;
    case OP_LE: return cmp_bytes(mn, lmn, lit, llit) <= 0;
    case OP_GT: return cmp_bytes(mx, lmx, lit, llit) > 0;
    default: return cmp_bytes(mx, lmx, lit, llit) >= 0;
  }
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

// native-width bits of row `row`, zero-extended
HORAE_HD uint64_t col_raw(const ColView& c, uint32_t row) {
  switch (c.width) {
    case 1: return reinterpret_cast<const uint8_t*>(c.vals)[row];
    case 2: return reinterpret_cast<const uint16_t*>(c.vals)[row];
    case 4: return reinterpret_cast<const uint32_t*>(c.vals)[row];
    default: return reinterpret_cast<const uint64_t*>(c.vals)[row];
  }
}

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

// Predicates on Binary columns (col.vals = one byte pointer per row, col.lens their lengths).  A literal carries its key (bytes_key).
struct BinLitDev { uint64_t key; const uint8_t* p; uint32_t len, _pad; };
struct BinPredDev {
  ColView col;
  uint32_t op, first, n_lit, _pad;   // literals [first, first + n_lit) of the set's table: 1 for a comparison, the list for OP_IN
};
struct BinPredSet { BinPredDev p[MAX_PREDS]; int n; uint32_t n_lits; const BinLitDev* lits; };
// OP_IN_SET predicates: keys[0 .. n) = the set's order keys, sorted and unique, in device memory
struct InSetDev { ColView col; const uint64_t* keys; uint32_t n, _pad; };
struct InSetPreds { InSetDev p[MAX_PREDS]; int n; };
struct PkSet { ColView c[MAX_PK]; int n; };

// 32-byte sort record of the k-way merge: (normalised PK : 128 bit, __seq__, row id) compared lexicographically.  `seq` is the
// value (0 when NULL); bit 32 of `row` is the value's validity, so that a NULL sorts before every value, u64 max included.
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

// Per-group counter partials (reduce_counter_groups_kernel).  first_* / last_* are the group's first / last row with a non-NULL value;
// valid[g] = 0 when it has none (then first_* / last_* are 0, increase 0.0 and resets 0).
struct CounterOut {
  void* gkey;            // native width of the group column
  int64_t* bucket;
  uint64_t* count;
  int64_t* first_ts;
  double* first_value;
  int64_t* last_ts;
  double* last_value;
  double* increase;
  uint64_t* resets;
  uint8_t* valid;        // one byte per group
};

}  // namespace horae
