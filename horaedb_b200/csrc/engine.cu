// engine.cu — host side of libhorae_gpu.so: SST residency, scan planning, pipeline orchestration, Arrow C export
// and the C ABI declared in include/horae_gpu.h.
//
// The planner mirrors ParquetReader::build_df_plan (read.rs:429-494):
//   ParquetExec (row-group pruning by chunk statistics)  -> FilterExec -> SortPreservingMergeExec -> MergeExec
// but runs every data-touching step as CUDA kernels (kernels.cu / fused_scan.cu).  There is no CPU fallback: if the
// device library cannot do something it returns HG_ERR_UNSUPPORTED.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "chunk_scratch.h"
#include "engine_internal.h"
#include "fused_scan.h"
#include "sst_writer.h"

thread_local Arena* g_arena = nullptr;
static thread_local std::string g_last_error;
int set_error(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

// A Snappy stream that holds only literals is the page's bytes behind a few header bytes: incompressible columns (random
// f64 values) are written as one literal per 64 KiB block.  A "stored" page is such a stream with at most two literals:
//   [varint: uncompressed size][literal 0 header][level prefix][first values][literal 1 header][the other values]
// Its layout as file offsets: literal i's bytes at lit[i] (len[1] = 0: one literal; literal 1's header starts at lit[0] + len[0]), and
// the bytes of the level prefix ([u32 len][RLE levels], optional columns only) at the start of literal 0.
struct StoredPage { uint64_t lit[2] = {0, 0}, len[2] = {0, 0}, prefix = 0; };
// Parses page pm as a stored page, with bounds checks; false when it is none
static bool stored_page(const uint8_t* data, uint64_t size, const PageMeta& pm, bool optional, StoredPage* sp) {
  const uint8_t* p = data + pm.payload_off;
  const uint8_t* end = p + pm.comp_size;
  if (pm.payload_off + pm.comp_size > size) return false;
  uint64_t ulen = 0;
  int sh = 0;
  for (;;) {
    if (p >= end || sh > 28) return false;
    const uint8_t b = *p++;
    ulen |= uint64_t(b & 0x7f) << sh;
    sh += 7;
    if (!(b & 0x80)) break;
  }
  if (ulen != pm.uncomp_size) return false;
  *sp = StoredPage();
  int n = 0;
  uint64_t total = 0;
  while (p < end) {
    if (n == 2) return false;
    const uint8_t t = *p;
    if (t & 3) return false;                       // a copy element: real compression
    uint64_t len = t >> 2;
    uint32_t hdr = 1;
    if (len >= 60) {
      const uint32_t nb = uint32_t(len) - 59;
      if (p + 1 + nb > end) return false;
      len = 0;
      for (uint32_t i = 0; i < nb; i++) len |= uint64_t(p[1 + i]) << (8 * i);
      hdr = 1 + nb;
    }
    len += 1;
    if (p + hdr + len > end) return false;
    sp->lit[n] = uint64_t(p + hdr - data);
    sp->len[n] = len;
    n++;
    total += len;
    p += hdr + len;
  }
  if (n == 0 || total != ulen) return false;
  if (optional) {
    if (sp->len[0] < 4) return false;
    uint32_t dl;
    std::memcpy(&dl, data + sp->lit[0], 4);
    sp->prefix = 4 + uint64_t(dl);
    if (sp->prefix > sp->len[0]) return false;
  }
  return true;
}

// True when the single V1 page of the chunk is a stored page whose literals both hold whole values, i.e. row i can be addressed in
// place: the fused scan then never decompresses the column.
static bool classify_stored(const uint8_t* data, uint64_t size, const PageMeta& pm, bool optional, uint32_t width, uint64_t rows) {
  StoredPage sp;
  if (!stored_page(data, size, pm, optional, &sp)) return false;
  if ((sp.len[0] - sp.prefix) % width != 0 || sp.len[1] % width != 0) return false;
  return sp.len[0] - sp.prefix + sp.len[1] == rows * width;
}

// Host-only, thread-safe: footer + page walk, validation against the schema, device tables, planning facts.
static int prepare_sst(const hg_schema_desc* schema, uint64_t id, const uint8_t* data, uint64_t size, SstResident* r,
                       std::vector<PageDev>* pages_out, std::vector<ChunkDev>* chunks_out, std::string* errmsg) {
  auto fail = [&](int code, const std::string& msg) { *errmsg = msg; return code; };
  r->id = id;
  r->size = size;
  std::string err;
  if (!parse_parquet(data, size, &r->meta, &err)) return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": " + err);
  const FileMetaData& m = r->meta;
  if (uint32_t(m.ncols) != schema->num_columns)
    return fail(HG_ERR_INVALID, "sst has " + std::to_string(m.ncols) + " columns, schema has " + std::to_string(schema->num_columns));
  for (int c = 0; c < m.ncols; c++) {
    if (m.phys_types[c] != phys_of(schema->types[c]))
      return fail(HG_ERR_INVALID, "column " + std::to_string(c) + ": parquet physical type does not match the schema");
    if (m.repetition[c] == 2) return fail(HG_ERR_UNSUPPORTED, "repeated columns");
  }
  std::vector<PageDev>& pages = *pages_out;
  pages.assign(m.pages.size(), PageDev());
  for (size_t i = 0; i < pages.size(); i++) {
    const PageMeta& pm = m.pages[i];
    if (pm.encoding != ENC_PLAIN && pm.encoding != ENC_DELTA_BINARY_PACKED && pm.encoding != ENC_DELTA_LENGTH_BYTE_ARRAY && pm.encoding != ENC_DELTA_BYTE_ARRAY &&
        pm.encoding != ENC_RLE_DICT && pm.encoding != ENC_PLAIN_DICT)
      return fail(HG_ERR_UNSUPPORTED, "page encoding " + std::to_string(pm.encoding) +
                                      " (PLAIN, DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY and RLE_DICTIONARY are implemented)");
    PageDev& pd = pages[i];
    pd.payload_off = pm.payload_off;
    pd.comp_size = pm.comp_size;
    pd.uncomp_size = pm.uncomp_size;
    pd.num_values = pm.num_values;
    pd.v2_def_len = pm.v2_def_len;
    pd.v2_rep_len = pm.v2_rep_len;
    pd.page_type = pm.page_type;
    pd.encoding = pm.encoding;
    pd.v2_compressed = pm.v2_compressed;
    pd._pad = 0;
  }
  std::vector<ChunkDev>& chunks = *chunks_out;
  chunks.assign(m.rgs.size() * size_t(m.ncols), ChunkDev());
  for (size_t g = 0; g < m.rgs.size(); g++)
    for (int c = 0; c < m.ncols; c++) {
      const ChunkMeta& cm = m.rgs[g].cols[c];
      if (cm.codec != CODEC_UNCOMPRESSED && cm.codec != CODEC_SNAPPY && cm.codec != CODEC_ZSTD)
        return fail(HG_ERR_UNSUPPORTED, "codec " + std::to_string(cm.codec) + " (UNCOMPRESSED, SNAPPY and ZSTD are implemented)");
      if (cm.scratch_bytes > 0xffffffffull) return fail(HG_ERR_UNSUPPORTED, "column chunk larger than 4 GiB");
      // the kernels decode by the CHUNK's physical type; the output buffers are laid out by the schema's
      if (cm.phys_type != m.phys_types[c])
        return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": column chunk type differs from the schema element's type");
      // every kernel indexes a chunk by the ROW GROUP's row count: the chunk must hold exactly that many values, and an
      // uncompressed page must really contain the bytes the decoders will read (compressed pages are bounded by their
      // scratch size on the device)
      if (cm.num_values != m.rgs[g].num_rows)
        return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": column chunk value count differs from the row group's row count");
      {
        const uint32_t pw = phys_width(cm.phys_type);
        const bool optional = m.repetition[c] == 1;
        const bool no_nulls = cm.phys_type != PT_BYTE_ARRAY && (!optional || (cm.stats.has_null_count && cm.stats.null_count == 0));   // (byte arrays: variable width)
        for (uint32_t pi = cm.first_page; pi < cm.first_page + cm.num_pages; pi++) {
          const PageMeta& pm = m.pages[pi];
          if (pm.page_type == PAGE_DATA_V2) {
            if (uint64_t(pm.v2_def_len) + pm.v2_rep_len > pm.comp_size || uint64_t(pm.v2_def_len) + pm.v2_rep_len > pm.uncomp_size)
              return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": V2 level bytes exceed the page");
            if (pm.encoding == ENC_PLAIN && no_nulls && uint64_t(pm.v2_def_len) + pm.v2_rep_len + uint64_t(pm.num_values) * pw > pm.uncomp_size)
              return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": page smaller than its values");
          } else if (cm.codec == CODEC_UNCOMPRESSED) {
            if (pm.comp_size != pm.uncomp_size) return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": uncompressed page with differing sizes");
            uint64_t prefix = 0;
            if (optional) {
              if (pm.uncomp_size < 4) return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": page smaller than its level header");
              uint32_t dl;
              std::memcpy(&dl, data + pm.payload_off, 4);
              prefix = 4 + uint64_t(dl);
              if (prefix > pm.uncomp_size) return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": definition levels exceed the page");
            }
            if (pm.encoding == ENC_PLAIN && no_nulls && prefix + uint64_t(pm.num_values) * pw > pm.uncomp_size)
              return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": page smaller than its values");
          }
        }
      }
      ChunkDev& cd = chunks[g * m.ncols + c];
      cd.first_page = cm.first_page;
      cd.num_pages = cm.num_pages;
      cd.scratch_bytes = uint32_t(cm.scratch_bytes);
      cd.phys = uint8_t(cm.phys_type);
      cd.codec = uint8_t(cm.codec);
      cd.optional = uint8_t(m.repetition[c] == 1);
      cd.stored = 0;
      // byte-array chunks take every encoding of the list above but DELTA_BINARY_PACKED, page by page (a dictionary chunk falls back to
      // PLAIN pages mid-chunk once its dictionary page is full).  The dictionary's entry count is the device's walk of the page; the
      // header's count must at least fit in it (4 bytes per entry)
      if (cm.phys_type == PT_BYTE_ARRAY && cm.has_dict_page && uint64_t(cm.dict_num_values) * 4 > cm.dict_uncomp_size)
        return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": byte-array dictionary page smaller than its entries");
      // an uncompressed dictionary page is read in place: it must not claim more bytes than it has
      if (cm.codec == CODEC_UNCOMPRESSED && cm.has_dict_page && cm.dict_comp_size != cm.dict_uncomp_size)
        return fail(HG_ERR_FORMAT, "sst " + std::to_string(id) + ": uncompressed dictionary page with differing sizes");
      cd.dict_payload_off = cm.has_dict_page ? cm.dict_payload_off : 0;
      cd.dict_comp = cm.has_dict_page ? cm.dict_comp_size : 0;
      cd.dict_uncomp = cm.has_dict_page ? cm.dict_uncomp_size : 0;
      for (uint32_t pi = cm.first_page; pi < cm.first_page + cm.num_pages; pi++) {
        if ((m.pages[pi].encoding == ENC_DELTA_LENGTH_BYTE_ARRAY || m.pages[pi].encoding == ENC_DELTA_BYTE_ARRAY) && cm.phys_type != PT_BYTE_ARRAY)
          return fail(HG_ERR_FORMAT, "DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY on a fixed-width column");
        if (m.pages[pi].encoding == ENC_DELTA_BINARY_PACKED && cm.phys_type != PT_INT32 && cm.phys_type != PT_INT64)
          return fail(HG_ERR_FORMAT, "DELTA_BINARY_PACKED on a non-integer column");
        if ((m.pages[pi].encoding == ENC_RLE_DICT || m.pages[pi].encoding == ENC_PLAIN_DICT) && !cm.has_dict_page)
          return fail(HG_ERR_FORMAT, "dictionary-encoded page without a dictionary page");
      }
      if (cm.phys_type != PT_BYTE_ARRAY && cm.codec == CODEC_SNAPPY && cm.num_pages == 1 && m.pages[cm.first_page].page_type == PAGE_DATA && m.rgs[g].num_rows > 0)
        cd.stored = classify_stored(data, size, m.pages[cm.first_page], cd.optional != 0, phys_width(cm.phys_type), uint64_t(m.rgs[g].num_rows)) ? 1 : 0;
    }
  r->rgcol.resize(m.rgs.size() * size_t(m.ncols));
  r->rg_rows.resize(m.rgs.size());
  for (size_t g = 0; g < m.rgs.size(); g++) {
    r->rg_rows[g] = uint32_t(m.rgs[g].num_rows);
    for (int c = 0; c < m.ncols; c++) {
      const ChunkMeta& cm = m.rgs[g].cols[c];
      RgCol& rc = r->rgcol[g * m.ncols + c];
      const uint32_t t = schema->types[c];
      if (cm.stats.has_min && cm.stats.has_max && cm.phys_type != PT_BYTE_ARRAY) {
        rc.has_minmax = 1;
        rc.mn = widen_stat(cm.stats.min, cm.phys_type, t);
        rc.mx = widen_stat(cm.stats.max, cm.phys_type, t);
      }
      rc.null_all = cm.stats.has_null_count && cm.stats.null_count == m.rgs[g].num_rows;
      rc.null_none = cm.stats.has_null_count && cm.stats.null_count == 0;
      rc.snappy = cm.codec == CODEC_SNAPPY;
      rc.scratch = uint32_t(cm.scratch_bytes);
      const bool one_plain_v1 = cm.num_pages == 1 && m.pages[cm.first_page].page_type == PAGE_DATA && m.pages[cm.first_page].encoding == ENC_PLAIN &&
                                !cm.has_dict_page && cm.phys_type != PT_BYTE_ARRAY;
      rc.single_page = one_plain_v1;
      rc.stored = chunks[g * m.ncols + c].stored;
      uint64_t boff = 0;
      uint32_t bbytes = 0;
      if (bloom_bitset(data, size, cm, &boff, &bbytes)) { rc.bloom_off = boff; rc.bloom_blocks = bbytes / 32; }
    }
  }
  {
    const uint32_t t0 = schema->types[0];
    for (int c = 0; c < m.ncols && c < MAX_COLS; c++) {
      r->col_null_none[c] = true; r->col_has_minmax[c] = true;
      r->col_all_single[c] = true; r->col_any_snappy[c] = false; r->col_snappy_all_stored[c] = true; r->col_snappy_any_stored[c] = false; r->col_any_zstd[c] = false;
    }
    for (size_t g = 0; g < m.rgs.size(); g++) {
      const uint32_t rows = r->rg_rows[g];
      r->rows_total += rows;
      if (rows == 0) continue;
      const RgCol* rc = &r->rgcol[g * m.ncols];
      for (int c = 0; c < m.ncols && c < MAX_COLS; c++) {
        if (!rc[c].single_page) r->col_all_single[c] = false;
        if (m.rgs[g].cols[c].codec == CODEC_ZSTD) { r->col_any_zstd[c] = true; r->any_zstd = true; }
        if (rc[c].snappy) { r->col_any_snappy[c] = true; if (!rc[c].stored) r->col_snappy_all_stored[c] = false; else r->col_snappy_any_stored[c] = true; }
        r->col_max_scratch[c] = std::max(r->col_max_scratch[c], rc[c].scratch);
        r->col_comp_bytes[c] += uint64_t(m.rgs[g].cols[c].total_compressed);
        if (!rc[c].null_none) r->col_null_none[c] = false;
        if (!rc[c].has_minmax) r->col_has_minmax[c] = false;
      }
      r->pk0.add(rc[0], t0);
      if (rc[0].has_minmax && rc[0].null_none) {
        uint64_t span = rc[0].mx - rc[0].mn + 1;
        r->group_bound += std::min<uint64_t>(span == 0 ? rows : span, rows) + 1;
      } else r->group_bound += uint64_t(rows) + 1;
    }
  }
  return HG_OK;
}

static int read_whole_file(const char* path, std::vector<uint8_t>* buf) {
  FILE* f = std::fopen(path, "rb");
  if (!f) return set_error(HG_ERR_NOT_FOUND, std::string("cannot open ") + path);
  long n = -1;
  if (std::fseek(f, 0, SEEK_END) == 0) n = std::ftell(f);
  if (n < 0 || std::fseek(f, 0, SEEK_SET) != 0) { std::fclose(f); return set_error(HG_ERR_NOT_FOUND, std::string("cannot size ") + path); }
  buf->resize(size_t(n));
  size_t got = std::fread(buf->data(), 1, size_t(n), f);
  std::fclose(f);
  if (got != size_t(n)) return set_error(HG_ERR_NOT_FOUND, std::string("short read on ") + path);
  return HG_OK;
}

// An SST parsed on the host: what prepare_sst makes of it, and the bytes it came from
struct ParsedSst {
  std::unique_ptr<SstResident> r;
  std::vector<PageDev> pages;
  std::vector<ChunkDev> chunks;
  std::vector<uint8_t> filebuf;      // the file's bytes, when they were read from hg_sst_desc::path
  const uint8_t* data = nullptr;     // the SST's bytes: the caller's, or filebuf
  uint64_t size = 0;
};

// The bytes of d (the caller's, or the file at d.path), parsed and validated against the schema; errors are reported through set_error
static int parse_sst(const hg_schema_desc* schema, const hg_sst_desc& d, ParsedSst* p) {
  p->data = d.data;
  p->size = d.size;
  if (!d.data) {
    if (!d.path) return set_error(HG_ERR_NOT_FOUND, "sst " + std::to_string(d.id) + ": neither data nor path given");
    int rc = read_whole_file(d.path, &p->filebuf);
    if (rc) return rc;
    p->data = p->filebuf.data();
    p->size = p->filebuf.size();
  }
  p->r = std::make_unique<SstResident>();
  std::string err;
  const int rc = prepare_sst(schema, d.id, p->data, p->size, p->r.get(), &p->pages, &p->chunks, &err);
  return rc ? set_error(rc, err) : HG_OK;
}

// One planning table of a file: the SstResident field that takes its device copy, its host source, its bytes and its allocation (at
// least one entry)
struct DevTable { void** dst; const void* src; size_t bytes, alloc; };
template <class T> static DevTable dev_table(T** dst, const std::vector<T>& v) {
  return DevTable{reinterpret_cast<void**>(dst), v.data(), v.size() * sizeof(T), std::max<size_t>(v.size(), 1) * sizeof(T)};
}
// The four planning tables of a parsed file: pages, chunks, rgcol and rg_rows.  In the device copy of rg_rows (*live_rows) a dead row
// group has zero rows, so every device-side planner prunes it.
static std::array<DevTable, 4> dev_tables(ParsedSst& p, std::vector<uint32_t>* live_rows) {
  SstResident& r = *p.r;
  live_rows->assign(r.rg_rows.begin(), r.rg_rows.end());
  for (size_t g = 0; g < r.rg_dead.size(); g++) if (r.rg_dead[g]) (*live_rows)[g] = 0;
  return {dev_table(&r.d_pages, p.pages), dev_table(&r.d_chunks, p.chunks), dev_table(&r.d_rgcol, r.rgcol), dev_table(&r.d_rg_rows, *live_rows)};
}

// hg_sst_load: the whole file becomes resident (cudaMalloc'd, cached until hg_sst_unload).
static int load_sst_locked(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* d) {
  if (e->ssts.count(d->id)) return HG_OK;
  ParsedSst p;
  int rc = parse_sst(schema, *d, &p);
  if (rc) return rc;
  std::vector<uint32_t> live_rows;
  const auto tables = dev_tables(p, &live_rows);
  uint64_t need = p.size + 64;
  for (const DevTable& t : tables) need += t.bytes;
  if (e->budget && e->resident_bytes + need > e->budget)
    return set_error(HG_ERR_OOM, "HBM budget exceeded while loading sst " + std::to_string(d->id));
  SstResident& r = *p.r;
  CU_TRY(cudaMalloc(&r.d_bytes, p.size + 64));
  for (const DevTable& t : tables) CU_TRY(cudaMalloc(t.dst, t.alloc));
  CU_TRY(cudaMemcpyAsync(r.d_bytes, p.data, p.size, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(cudaMemsetAsync(r.d_bytes + p.size, 0, 64, e->stream));
  for (const DevTable& t : tables) if (t.bytes) CU_TRY(cudaMemcpyAsync(*t.dst, t.src, t.bytes, cudaMemcpyHostToDevice, e->stream));
  CU_TRY(cudaStreamSynchronize(e->stream));
  r.device_bytes = need;
  e->resident_bytes += need;
  e->stats.bytes_h2d += need;
  e->ssts[d->id] = std::move(p.r);
  return HG_OK;
}

// ------------------------------------------------------------------------------------------------------ scan planning
// Sorted, unique order keys of every HG_OP_IN_SET predicate's values.  An index lookup usually delivers its ids in order: one pass checks
// for "strictly increasing" while converting, and only a set that is not gets sorted.
void prepare_in_sets(const hg_schema_desc* schema, const hg_predicate* preds, size_t np, InSets* out) {
  for (size_t i = 0; i < size_t(MAX_PREDS); i++) {
    std::vector<uint64_t>& keys = out->keys[i];
    keys.clear();
    if (i >= np || preds[i].op != HG_OP_IN_SET) continue;
    const auto t0 = HostClock::now();
    const uint64_t flip = order_flip(schema->types[preds[i].column]);
    const uint32_t n = preds[i].in_count;
    keys.resize(n);
    bool increasing = true;
    for (uint32_t j = 0; j < n; j++) {
      keys[j] = preds[i].in_values[j] ^ flip;
      if (j && keys[j] <= keys[j - 1]) increasing = false;
    }
    if (!increasing) {
      std::sort(keys.begin(), keys.end());
      keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    }
    if (trace_on())
      fprintf(stderr, "[in_set] predicate %zu: %u values -> %zu keys, %s, %.0f us\n", i, n, keys.size(), increasing ? "already sorted" : "sorted on the host",
              elapsed_us(t0, HostClock::now()));
  }
}

static bool rg_may_match(const SstResident& f, size_t g, const hg_schema_desc* schema, const hg_predicate* preds, const uint64_t* lits, size_t np,
                         const InSets& sets) {
  // DataFusion PruningPredicate (pinned by the plan text at read.rs:613):
  //   CASE WHEN null_count = row_count THEN false ELSE <min/max rewrite of the comparison> END
  const RgCol* rc = &f.rgcol[g * size_t(f.meta.ncols)];
  for (size_t i = 0; i < np; i++) {
    const RgCol& c = rc[preds[i].column];
    const uint32_t t = schema->types[preds[i].column];
    const uint32_t cls = cmp_class(t);
    if (c.null_all) return false;
    bool ok;
    if (t == T_BINARY) {              // the chunk's whole min_value / max_value, kept on the host (never in RgCol)
      const ColumnStats& st = f.meta.rgs[g].cols[preds[i].column].stats;
      if (!st.has_bin_min || !st.has_bin_max) continue;
      const uint8_t* sb = f.meta.stat_bytes.data();
      const bool in = preds[i].op == HG_OP_IN;
      ok = false;
      for (uint32_t j = 0; j < (in ? preds[i].in_count : 1u) && !ok; j++)
        ok = bytes_minmax_may_match(sb + st.bin_min_off, st.bin_min_len, sb + st.bin_max_off, st.bin_max_len, preds[i].in_bytes[j].data,
                                    preds[i].in_bytes[j].len, in ? uint32_t(OP_EQ) : preds[i].op);
      if (!ok) return false;
      continue;
    }
    if (!c.has_minmax) continue;
    if (preds[i].op == HG_OP_IN) {    // PruningPredicate expands a short IN list into `c = v1 OR c = v2 ..`
      ok = false;
      for (uint32_t j = 0; j < preds[i].in_count && !ok; j++) ok = minmax_may_match(c.mn, c.mx, preds[i].in_values[j], OP_EQ, cls);
    } else if (preds[i].op == HG_OP_IN_SET) {   // the same rewrite for a set of any size: some member inside [min, max]
      uint32_t lo, hi;
      ok = key_set_slice(sets.keys[i].data(), uint32_t(sets.keys[i].size()), order_key(c.mn, t), order_key(c.mx, t), &lo, &hi);
    } else ok = minmax_may_match(c.mn, c.mx, lits[i], preds[i].op, cls);
    if (!ok) return false;
  }
  return true;
}

// Whether row group g of a parsed file may hold a row passing the predicates, on the host: it has rows, its statistics admit the
// predicates (not tested when np = 0) and its bloom filters do not rule them out (not probed when bl.n = 0)
static bool rg_survives(const ParsedSst& f, size_t g, const hg_schema_desc* schema, const hg_predicate* preds, const uint64_t* lits, size_t np,
                        const InSets& sets, const BloomLits& bl) {
  const SstResident& r = *f.r;
  if (r.rg_rows[g] == 0) return false;
  if (np && !rg_may_match(r, g, schema, preds, lits, np, sets)) return false;
  return !bl.n || bloom_may_match_host(&r.rgcol[g * size_t(r.meta.ncols)], f.data, bl);
}

// Small host -> device uploads go through one pinned staging buffer.  The cursor is per CALL (reset in reset_call, when the
// stream is idle): copies are asynchronous, so a region must not be reused before the stream has consumed it.
int stage_upload(hg_engine* e, void* dst, const void* src, size_t bytes) {
  size_t off = (e->stage_cursor + 255) & ~size_t(255);
  if (off + bytes > e->h_stage_bytes) {
    // grow (rare): everything staged so far in this call must reach the device first
    CU_TRY(cudaStreamSynchronize(e->stream));
    size_t nb = std::max<size_t>((off + bytes) * 2, 1 << 20);
    void* p = nullptr;
    CU_TRY(cudaMallocHost(&p, nb));
    if (e->h_stage) cudaFreeHost(e->h_stage);
    e->h_stage = p;
    e->h_stage_bytes = nb;
    off = 0;
  }
  std::memcpy(static_cast<char*>(e->h_stage) + off, src, bytes);
  CU_TRY(cudaMemcpyAsync(dst, static_cast<char*>(e->h_stage) + off, bytes, cudaMemcpyHostToDevice, e->stream));
  e->stage_cursor = off + bytes;
  return HG_OK;
}


// ------------------------------------------------------------------------------------- transient, selective SST loads
// A scan called with host bytes for SSTs that are not resident does not cache them: it copies ONLY the byte ranges the
// query can touch — column chunks of the needed columns in row groups that survive statistics pruning — into arena
// memory laid out at the file's own offsets (so the page table stays valid), uploads the page tables, and forgets
// everything at the end of the call.  Footers are parsed on a small thread pool.  With pinned host buffers the ranges
// are fetched by one gather kernel reading host memory over PCIe (no per-range API call).
struct CopyRange { const uint8_t* src; uint8_t* dst; uint64_t bytes; };

__global__ void __launch_bounds__(256) gather_ranges_kernel(const CopyRange* __restrict__ ranges, uint32_t nranges) {
  for (uint32_t r = blockIdx.x; r < nranges; r += gridDim.x) {
    const CopyRange cr = ranges[r];
    const uintptr_t sa = reinterpret_cast<uintptr_t>(cr.src), da = reinterpret_cast<uintptr_t>(cr.dst);
    if (((sa ^ da) & 15) == 0) {
      uint64_t head = (16 - (sa & 15)) & 15;
      if (head > cr.bytes) head = cr.bytes;
      for (uint64_t i = threadIdx.x; i < head; i += 256) cr.dst[i] = cr.src[i];
      const uint64_t nvec = (cr.bytes - head) >> 4;
      const uint4* s = reinterpret_cast<const uint4*>(cr.src + head);
      uint4* d = reinterpret_cast<uint4*>(cr.dst + head);
      for (uint64_t i = threadIdx.x; i < nvec; i += 256) d[i] = s[i];
      for (uint64_t i = head + (nvec << 4) + threadIdx.x; i < cr.bytes; i += 256) cr.dst[i] = cr.src[i];
    } else {
      for (uint64_t i = threadIdx.x; i < cr.bytes; i += 256) cr.dst[i] = cr.src[i];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- host worker pool
// A transient load parses footers / page headers and builds tens of thousands of byte ranges per call on the host while PCIe waits:
// per-file work, run on a small persistent pool (threads created per call cost as much as the work they would do).
namespace {
class WorkPool {
 public:
  explicit WorkPool(unsigned n) { for (unsigned i = 0; i < n; i++) th_.emplace_back([this] { loop(); }); }
  ~WorkPool() {
    { std::lock_guard<std::mutex> g(mu_); stop_ = true; }
    cv_.notify_all();
    for (auto& t : th_) t.join();
  }
  // fn(i) for every i in [0, n), on the workers and on the caller; returns when all have finished
  void parallel_for(size_t n, const std::function<void(size_t)>& fn) {
    if (n == 0) return;
    if (n == 1 || th_.empty()) { for (size_t i = 0; i < n; i++) fn(i); return; }
    std::lock_guard<std::mutex> serial(call_mu_);           // one parallel_for at a time
    {
      std::lock_guard<std::mutex> g(mu_);
      fn_ = &fn; n_ = n; next_.store(0); done_ = 0; gen_++;
    }
    cv_.notify_all();
    run();
    std::unique_lock<std::mutex> g(mu_);
    cv_done_.wait(g, [&] { return done_ == n_; });
    fn_ = nullptr;
  }

 private:
  void run() {
    size_t mine = 0;
    for (;;) {
      const size_t i = next_.fetch_add(1);
      if (i >= n_) break;
      (*fn_)(i);
      mine++;
    }
    if (mine) {
      std::lock_guard<std::mutex> g(mu_);
      done_ += mine;
      if (done_ == n_) cv_done_.notify_all();
    }
  }
  void loop() {
    uint64_t seen = 0;
    for (;;) {
      {
        std::unique_lock<std::mutex> g(mu_);
        cv_.wait(g, [&] { return stop_ || gen_ != seen; });
        if (stop_) return;
        seen = gen_;
      }
      run();
    }
  }
  std::vector<std::thread> th_;
  std::mutex mu_, call_mu_;
  std::condition_variable cv_, cv_done_;
  const std::function<void(size_t)>* fn_ = nullptr;
  size_t n_ = 0, done_ = 0;
  std::atomic<size_t> next_{0};
  uint64_t gen_ = 0;
  bool stop_ = false;
};
WorkPool& work_pool() {
  static WorkPool* p = new WorkPool(std::min(15u, std::max(1u, std::thread::hardware_concurrency() / 2)));   // + the caller = 16
  return *p;
}
}  // namespace

// File f's byte range [lo, hi), merged into the previous range of the list when they touch
static void add_bytes(std::vector<CopyRange>* ranges, const ParsedSst& f, uint64_t lo, uint64_t hi) {
  const SstResident& r = *f.r;
  hi = std::min<uint64_t>(r.size, hi + 16);               // the unaligned 8-byte loads may touch one word past the values
  if (lo >= hi) return;
  CopyRange* b = ranges->empty() ? nullptr : &ranges->back();
  if (b && b->src + b->bytes >= f.data + lo && b->src <= f.data + lo && b->dst == r.d_bytes + (b->src - f.data))
    b->bytes = std::max<uint64_t>(uint64_t(b->src - f.data) + b->bytes, hi) - uint64_t(b->src - f.data);
  else ranges->push_back(CopyRange{f.data + lo, r.d_bytes + lo, hi - lo});
}

// The whole column chunk (g, c), from its dictionary page when it has one
static void add_chunk(std::vector<CopyRange>* ranges, const ParsedSst& f, uint32_t g, uint32_t c) {
  const ChunkMeta& cm = f.r->meta.rgs[g].cols[c];
  uint64_t lo = uint64_t(cm.data_page_offset);
  if (cm.dict_page_offset > 0 && uint64_t(cm.dict_page_offset) < lo) lo = uint64_t(cm.dict_page_offset);
  add_bytes(ranges, f, lo, lo + uint64_t(cm.total_compressed));
}

// A Snappy page the device will decode only up to the last gate-passing row (fused scan, partial decode) travels as a PREFIX of its
// compressed stream: the share of the stream that the needed share of the output takes, plus a margin.  The page table tells the
// decoder where the prefix ends; a stream that turns out lopsided ends early, the decoder reports it, and the entry point repeats the
// call without prefixes (e->trunc_used) — never a wrong result.  False, and nothing added, when the prefix would save too little.
static bool add_prefix(std::vector<CopyRange>* ranges, ParsedSst& f, uint32_t g, uint32_t c, uint32_t last) {
  const ChunkDev& cd = f.chunks[size_t(g) * size_t(f.r->meta.ncols) + c];
  PageDev& pg = f.pages[cd.first_page];
  const uint32_t w = phys_width(cd.phys);
  const uint64_t rows = f.r->rg_rows[g];
  const uint64_t out_row = std::min<uint64_t>(uint64_t(last) + 2, rows);             // gate_rg_kernel's RgSel::out_row
  const uint64_t need_uncomp = 16 + (rows + 7) / 8 + 8 + out_row * w + 2304;        // stop_at + one batch of overshoot
  const uint64_t est = uint64_t(double(pg.comp_size) * double(need_uncomp) / double(std::max<uint32_t>(pg.uncomp_size, 1)) * 1.08) + 1024;
  if (est + 4096 >= pg.comp_size) return false;
  add_bytes(ranges, f, uint64_t(f.r->meta.rgs[g].cols[c].data_page_offset), pg.payload_off + est);
  pg.comp_size = uint32_t(est);
  return true;
}

// A page whose values can be addressed by row (uncompressed PLAIN, or stored Snappy: sp): its level prefix, and of its values only the
// blocks of rows that hold a passing row (GateOut::mask), cut to [first, last]; adjacent blocks travel as one interval
static void add_row_window(std::vector<CopyRange>* ranges, const ParsedSst& f, uint32_t g, const ChunkDev& cd, const StoredPage& sp,
                           const fused::GateOut& go) {
  const uint32_t w = phys_width(cd.phys);
  const uint64_t body = f.pages[cd.first_page].payload_off;
  // layout: PLAIN page = [prefix][values]; stored page = see StoredPage
  uint64_t v0 = body, v1 = 0, n0 = ~0ull;                               // v0 / v1: file offsets of value 0 and of value n0
  if (cd.codec == CODEC_UNCOMPRESSED) {
    uint64_t prefix = 0;
    if (cd.optional) { uint32_t dl; std::memcpy(&dl, f.data + body, 4); prefix = 4 + uint64_t(dl); }
    add_bytes(ranges, f, body, body + prefix);
    v0 = body + prefix;
  } else {
    n0 = (sp.len[0] - sp.prefix) / w;
    add_bytes(ranges, f, body, sp.lit[0] + sp.prefix);
    v0 = sp.lit[0] + sp.prefix;
    if (sp.len[1]) {
      v1 = sp.lit[1];
      add_bytes(ranges, f, sp.lit[0] + sp.len[0], v1);
    }
  }
  const uint32_t brows = fused::gate_block_rows(f.r->rg_rows[g]);
  for (uint32_t b = 0; b < 32u;) {
    if (!((go.mask >> b) & 1u)) { b++; continue; }
    uint32_t e2 = b;
    while (e2 + 1 < 32u && ((go.mask >> (e2 + 1)) & 1u)) e2++;
    const uint64_t first = std::max<uint64_t>(go.first, uint64_t(b) * brows);
    const uint64_t last = std::min<uint64_t>(go.last, uint64_t(e2 + 1) * brows - 1);
    b = e2 + 1;
    if (first > last) continue;
    if (first < n0) add_bytes(ranges, f, v0 + first * w, v0 + (std::min<uint64_t>(last, n0 - 1) + 1) * w);
    if (v1 && last >= n0) add_bytes(ranges, f, v1 + (std::max<uint64_t>(first, n0) - n0) * w, v1 + (last - n0 + 1) * w);
  }
}

// Late materialisation across PCIe: the gate column is a predicate column that is one PLAIN page without NULLs in every chunk of every
// file (Snappy or not) and has no IN / IN_SET predicate (the gate kernel tests intervals); the one with the fewest compressed bytes, unless
// those are most of the needed bytes anyway.  -1: no gate.
static int choose_gate_col(const std::vector<ParsedSst>& files, const hg_predicate* preds, size_t np, const std::vector<uint32_t>& need_cols) {
  int gate_col = -1;
  uint64_t best_bytes = ~0ull;
  for (size_t i = 0; i < np; i++) {
    const uint32_t c = preds[i].column;
    bool ok = c < uint32_t(MAX_COLS);
    for (size_t i2 = 0; i2 < np; i2++)
      if (preds[i2].column == c && (preds[i2].op == HG_OP_IN || preds[i2].op == HG_OP_IN_SET)) ok = false;
    uint64_t bytes = 0;
    for (size_t j = 0; j < files.size() && ok; j++) {
      const SstResident& r = *files[j].r;
      ok = r.rows_total == 0 || r.row_addressable(c);
      bytes += r.col_comp_bytes[c];
    }
    if (ok && bytes < best_bytes) { best_bytes = bytes; gate_col = int(c); }
  }
  uint64_t need_bytes = 0;
  for (uint32_t c : need_cols) for (const ParsedSst& f : files) need_bytes += f.r->col_comp_bytes[c];
  return gate_col >= 0 && best_bytes * 2 > need_bytes ? -1 : gate_col;
}

// The gate column of one file's kept row groups, built on the worker pool: its byte ranges, its Snappy pages (decompressed on the
// device into scratch `scratch` bytes into the file's share, allocated once the pool is done) and the gate descriptors
struct GateFile {
  struct SnappyPage { size_t i; uint64_t scratch; k::RawPage raw; };   // i: index into kept[]; raw.dst is set with the scratch
  std::vector<CopyRange> ranges;
  std::vector<SnappyPage> snappy;
  uint64_t scratch_bytes = 0;
  int code = HG_OK;
  std::string err;
};

// One transient load.  kept[] lists the row groups the host keeps, ordered by file (seg[j] = file j's [begin, end) of it); every other
// row group of a file is dead (SstResident::rg_dead).  With a gate column, gate_out[i] is the gate's result for kept[i].
struct TransientLoad {
  struct KeptRg { uint32_t j, g; };
  hg_engine* e;
  const hg_schema_desc* schema;
  const hg_predicate* preds;
  size_t np;
  std::vector<uint32_t> need_cols;
  std::vector<ParsedSst> files;
  std::vector<KeptRg> kept;
  std::vector<std::pair<size_t, size_t>> seg;
  int gate_col = -1;
  std::vector<fused::GateOut> gate_out;
  bool all_pinned = false;
  uint64_t copied = 0;
  size_t n_ranges = 0;

  // Moves a batch of byte ranges host -> device on the engine's stream: one gather kernel when every file's bytes are pinned
  int move_ranges(std::vector<CopyRange>& ranges) {
    n_ranges += ranges.size();
    for (auto& cr : ranges) copied += cr.bytes;
    if (ranges.empty()) return HG_OK;
    if (all_pinned) {
      CopyRange* d_ranges = static_cast<CopyRange*>(g_arena->alloc(ranges.size() * sizeof(CopyRange)));
      if (!d_ranges) return set_error(HG_ERR_OOM, "out of device memory");
      int rc = stage_upload(e, d_ranges, ranges.data(), ranges.size() * sizeof(CopyRange));
      if (rc) return rc;
      gather_ranges_kernel<<<int(std::min<size_t>(ranges.size(), kNumSMs * 8)), 256, 0, e->stream>>>(d_ranges, uint32_t(ranges.size()));
      e->launches++;
    } else {
      for (auto& cr : ranges) CU_TRY(cudaMemcpyAsync(cr.dst, cr.src, cr.bytes, cudaMemcpyHostToDevice, e->stream));
    }
    return HG_OK;
  }

  // Parses the files on the worker pool; adds __seq__ to the needed columns unless the inputs are provably PK-disjoint (then no real
  // merge runs); gives every file its image in arena memory, at the file's own offsets so that the page table stays valid
  int parse(const hg_sst_desc* ssts, const std::vector<size_t>& pending, bool seq_if_overlap, const std::vector<size_t>& resident_idx) {
    const size_t nf = pending.size();
    files.resize(nf);
    std::vector<int> codes(nf, HG_OK);
    std::vector<std::string> errs(nf);
    work_pool().parallel_for(nf, [&](size_t j) {
      codes[j] = parse_sst(schema, ssts[pending[j]], &files[j]);
      if (codes[j]) errs[j] = g_last_error;                 // set_error's message is per thread
    });
    for (size_t j = 0; j < nf; j++) if (codes[j]) return set_error(codes[j], errs[j]);
    if (seq_if_overlap) {
      std::vector<Pk0Range> all;
      for (const ParsedSst& f : files) if (f.r->rows_total) all.push_back(f.r->pk0);
      for (size_t i : resident_idx) { auto it = e->ssts.find(ssts[i].id); if (it != e->ssts.end() && it->second->rows_total) all.push_back(it->second->pk0); }
      std::vector<size_t> order;
      if (all.size() > 1 && !pk0_disjoint(all, schema->types[0], &order)) need_cols.push_back(schema->num_columns - 2);
    }
    std::sort(need_cols.begin(), need_cols.end());
    need_cols.erase(std::unique(need_cols.begin(), need_cols.end()), need_cols.end());
    all_pinned = nf > 0;
    for (size_t j = 0; j < nf && all_pinned; j++) {
      cudaPointerAttributes at;
      if (cudaPointerGetAttributes(&at, files[j].data) != cudaSuccess || at.type != cudaMemoryTypeHost) { all_pinned = false; cudaGetLastError(); }
    }
    for (ParsedSst& f : files) {
      SstResident& r = *f.r;
      r.owned = false;
      r.rg_dead.assign(r.rg_rows.size(), 0);
      r.d_bytes = static_cast<uint8_t*>(g_arena->alloc(r.size + 64));
      if (!r.d_bytes) return set_error(HG_ERR_OOM, "out of device memory for transient SST");
    }
    return HG_OK;
  }

  // The row groups that survive statistics and bloom-filter pruning.  The filters are probed here, in host memory: they never cross
  // PCIe, so the device tables of a transient file list none
  void keep_row_groups() {
    const bool prune = !(e->flags & HG_FLAG_NO_PRUNING);
    uint64_t lits[MAX_PREDS];
    for (size_t i = 0; i < np; i++) lits[i] = pred_literal(preds[i], schema->types[preds[i].column]);
    BloomLits bl;
    if (prune && np && !(e->flags & HG_FLAG_NO_BLOOM_FILTER)) bloom_literals(schema, preds, np, &bl);
    seg.assign(files.size(), {0, 0});
    for (size_t j = 0; j < files.size(); j++) {
      SstResident& r = *files[j].r;
      const size_t ncols = size_t(r.meta.ncols);
      seg[j].first = kept.size();
      for (size_t g = 0; g < r.rg_rows.size(); g++) {
        if (rg_survives(files[j], g, schema, preds, lits, prune ? np : 0, e->in_sets, bl)) kept.push_back(KeptRg{uint32_t(j), uint32_t(g)});
        else r.rg_dead[g] = 1;
        for (size_t c = 0; c < ncols; c++) r.rgcol[g * ncols + c].bloom_blocks = 0;
      }
      seg[j].second = kept.size();
    }
  }

  // File j's share of the gate phase (worker pool)
  void gate_file(size_t j, fused::GateRg* descs, GateFile* gf) const {
    const ParsedSst& f = files[j];
    const SstResident& r = *f.r;
    const uint32_t gw = type_width(schema->types[gate_col]) <= 4 ? 4u : 8u;
    auto fail = [&](const char* msg) { gf->code = HG_ERR_FORMAT; gf->err = msg; };
    for (size_t i = seg[j].first; i < seg[j].second; i++) {
      const uint32_t g = kept[i].g, rows = r.rg_rows[g];
      add_chunk(&gf->ranges, f, g, uint32_t(gate_col));
      const ChunkDev& cd = f.chunks[size_t(g) * size_t(r.meta.ncols) + size_t(gate_col)];
      const PageDev& pg = f.pages[cd.first_page];
      uint64_t off = pg.payload_off;
      if (cd.codec == CODEC_SNAPPY) {                       // decompressed on the device; the level prefix is skipped there
        gf->snappy.push_back(GateFile::SnappyPage{i, gf->scratch_bytes, k::RawPage{r.d_bytes + off, nullptr, pg.comp_size, pg.uncomp_size}});
        gf->scratch_bytes += (scratch_region(pg.uncomp_size) + 16 + 255) & ~uint64_t(255);
        if (uint64_t(pg.uncomp_size) < uint64_t(rows) * gw) return fail("column chunk smaller than its values");
        descs[i] = fused::GateRg{nullptr, rows, cd.optional ? 1u : 0u};
      } else {
        if (cd.optional) {                                  // [u32 len][RLE def levels] in front of the values (all valid here)
          uint32_t len = 0;
          if (off + 4 > r.size) return fail("page payload out of bounds");
          std::memcpy(&len, f.data + off, 4);
          off += 4 + uint64_t(len);
        }
        if (off + uint64_t(rows) * gw > r.size) return fail("column chunk out of bounds");
        descs[i] = fused::GateRg{r.d_bytes + off, rows, 0};
      }
    }
  }

  // The gate column's chunks move first; the device finds, per kept row group, the first and the last row that pass the predicates on
  // that column, and a row group with none becomes dead.  The filter precedes merge and dedup (read.rs:459-480): rows that fail the
  // gate take part in nothing downstream.
  int run_gate() {
    std::vector<fused::GateRg> descs(kept.size());
    std::vector<GateFile> gfs(files.size());
    work_pool().parallel_for(files.size(), [&](size_t j) { gate_file(j, descs.data(), &gfs[j]); });
    std::vector<k::RawPage> raw;
    for (GateFile& gf : gfs) {
      if (gf.code) return set_error(gf.code, gf.err);
      uint8_t* base = nullptr;
      if (gf.scratch_bytes) {
        base = static_cast<uint8_t*>(g_arena->alloc(gf.scratch_bytes));
        if (!base) return set_error(HG_ERR_OOM, "out of device memory");
      }
      for (GateFile::SnappyPage& sp : gf.snappy) {
        sp.raw.dst = base + sp.scratch;
        descs[sp.i].vals = sp.raw.dst;
        raw.push_back(sp.raw);
      }
      int rc = move_ranges(gf.ranges);
      if (rc) return rc;
    }
    fused::GateRg* d_descs = static_cast<fused::GateRg*>(g_arena->alloc(descs.size() * sizeof(fused::GateRg)));
    fused::GateOut* d_out = static_cast<fused::GateOut*>(g_arena->alloc(kept.size() * sizeof(fused::GateOut) + 16));
    uint32_t* d_tick = static_cast<uint32_t*>(g_arena->alloc(64));
    if (!d_descs || !d_out || !d_tick) return set_error(HG_ERR_OOM, "out of device memory");
    CU_TRY(cudaMemsetAsync(d_tick, 0, 64, e->stream));
    int rc = 0;
    if (!raw.empty()) {
      k::RawPage* d_raw = static_cast<k::RawPage*>(g_arena->alloc(raw.size() * sizeof(k::RawPage)));
      if (!d_raw) return set_error(HG_ERR_OOM, "out of device memory");
      rc = stage_upload(e, d_raw, raw.data(), raw.size() * sizeof(k::RawPage));
      if (rc) return rc;
      k::snappy_raw_pages(e->L(), d_raw, uint32_t(raw.size()), d_tick, reinterpret_cast<int*>(d_tick + 1));
    }
    rc = stage_upload(e, d_descs, descs.data(), descs.size() * sizeof(fused::GateRg));
    if (rc) return rc;
    hg_predicate gp[MAX_PREDS];
    size_t ngp = 0;
    for (size_t i = 0; i < np; i++) if (int(preds[i].column) == gate_col) gp[ngp++] = preds[i];
    rc = fused::gate_row_groups(e, d_descs, uint32_t(kept.size()), schema->types[gate_col], gp, ngp, d_out);
    if (rc) return rc;
    gate_out.resize(kept.size());
    int herr = 0;
    CU_TRY(cudaMemcpyAsync(gate_out.data(), d_out, kept.size() * sizeof(fused::GateOut), cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(&herr, d_tick + 1, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    if (herr) return set_error(HG_ERR_FORMAT, "device decode error code " + std::to_string(herr) + " (gate column)");
    e->stats.bytes_d2h += kept.size() * sizeof(fused::GateOut);
    e->stage_cursor = 0;                                    // the stream is idle: the staging buffer can be reused
    for (size_t i = 0; i < kept.size(); i++)
      if (gate_out[i].first > gate_out[i].last) files[kept[i].j].r->rg_dead[kept[i].g] = 1;
    return HG_OK;
  }

  // File j's byte ranges of the needed columns, the gate column excluded, in its live row groups (worker pool).  After a gate, the
  // non-key columns that can be addressed by row move only the rows the gate found, and the Snappy pages decoded up to the last
  // gate-passing row only a prefix; true when some page travels as such a prefix.
  bool file_ranges(size_t j, std::vector<CopyRange>* ranges) {
    ParsedSst& f = files[j];
    const SstResident& r = *f.r;
    const bool gated = gate_col >= 0, prefixes = gated && gate_col == e->trunc_gate;
    bool trunc = false;
    for (size_t i = seg[j].first; i < seg[j].second; i++) {
      const uint32_t g = kept[i].g;
      if (r.rg_dead[g]) continue;
      for (uint32_t c : need_cols) {
        if (int(c) == gate_col) continue;
        const ChunkDev& cd = f.chunks[size_t(g) * size_t(r.meta.ncols) + c];
        const RgCol& rc = r.rgcol[size_t(g) * size_t(r.meta.ncols) + c];
        StoredPage sp;
        if (gated && c >= schema->num_primary_keys && rc.single_page && rc.null_none &&
            (cd.codec == CODEC_UNCOMPRESSED || (cd.stored && stored_page(f.data, r.size, r.meta.pages[cd.first_page], cd.optional, &sp))))
          add_row_window(ranges, f, g, cd, sp, gate_out[i]);
        else if (prefixes && c < 32 && ((e->trunc_mask >> c) & 1u) && cd.codec == CODEC_SNAPPY && rc.single_page && !cd.stored &&
                 add_prefix(ranges, f, g, c, gate_out[i].last))
          trunc = true;
        else
          add_chunk(ranges, f, g, c);
      }
    }
    return trunc;
  }

  // The main transfer: one task per file on the worker pool (a file's ranges only touch that file's tables); the files' range lists
  // leave in file order
  int move_main_ranges() {
    std::vector<std::vector<CopyRange>> ranges(files.size());
    std::vector<uint8_t> trunc(files.size(), 0);
    work_pool().parallel_for(files.size(), [&](size_t j) { trunc[j] = file_ranges(j, &ranges[j]) ? 1 : 0; });
    for (size_t j = 0; j < files.size(); j++) {
      if (trunc[j]) e->trunc_used = true;
      int rc = move_ranges(ranges[j]);
      if (rc) return rc;
    }
    return HG_OK;
  }

  // The planning tables in arena memory.  bytes_h2d counts a transient file's pages, chunks and rgcol, not its rg_rows.
  int upload_tables() {
    for (ParsedSst& f : files) {
      std::vector<uint32_t> live_rows;
      const auto tables = dev_tables(f, &live_rows);
      for (const DevTable& t : tables) {
        if (!(*t.dst = g_arena->alloc(t.alloc))) return set_error(HG_ERR_OOM, "out of device memory for transient SST");
        int rc = t.bytes ? stage_upload(e, *t.dst, t.src, t.bytes) : HG_OK;
        if (rc) return rc;
      }
      copied += tables[0].bytes + tables[1].bytes + tables[2].bytes;
    }
    e->stats.bytes_h2d += copied;
    return HG_OK;
  }

  // The files join e->ssts until the end of the call
  int commit() {
    bool from_path = false;
    for (ParsedSst& f : files) {
      from_path = from_path || !f.filebuf.empty();
      e->transient_ids.push_back(f.r->id);
      e->ssts[f.r->id] = std::move(f.r);
    }
    // host buffers read from files must outlive the async copies
    if (!all_pinned || from_path) CU_TRY(cudaStreamSynchronize(e->stream));
    return HG_OK;
  }
};

// A call's SSTs that are not resident: only the byte ranges the call can touch cross PCIe (see TransientLoad)
static int load_transient(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, const std::vector<size_t>& pending,
                          const hg_predicate* preds, size_t np, std::vector<uint32_t> need_cols, bool seq_if_overlap,
                          const std::vector<size_t>& resident_idx) {
  TransientLoad t{e, schema, preds, np, std::move(need_cols)};
  const auto t0 = HostClock::now();
  int rc = t.parse(ssts, pending, seq_if_overlap, resident_idx);
  if (rc) return rc;
  const auto t1 = HostClock::now();
  t.keep_row_groups();
  if (!(e->flags & (HG_FLAG_NO_PRUNING | HG_FLAG_NO_LATE_MATERIALIZATION)) && np && t.need_cols.size() > 1 && !t.kept.empty())
    t.gate_col = choose_gate_col(t.files, preds, np, t.need_cols);
  if (t.gate_col >= 0 && (rc = t.run_gate())) return rc;
  const auto t2 = HostClock::now();
  if ((rc = t.move_main_ranges())) return rc;
  const auto t3 = HostClock::now();
  if ((rc = t.upload_tables())) return rc;
  if (trace_on()) {
    const auto t4 = HostClock::now();
    cudaStreamSynchronize(e->stream);
    fprintf(stderr, "[transient] %zu files: parse %.0f us, gate phase %.0f us, main ranges %.0f us, tables %.0f us (%zu ranges, %.1f MB, gate column %d), copy wait %.0f us\n",
            t.files.size(), elapsed_us(t0, t1), elapsed_us(t1, t2), elapsed_us(t2, t3), elapsed_us(t3, t4), t.n_ranges, t.copied / 1e6, t.gate_col,
            elapsed_us(t4, HostClock::now()));
  }
  return t.commit();
}

namespace {
struct FileSel { SstResident* f; std::vector<uint32_t> rgs; };

// One (row group, `=` / `IN` predicate) pair to probe: the bitset inside the resident file bytes and the predicate's literal hashes
struct BloomProbeDev { const uint8_t* bits; uint32_t nblocks, first, count, _pad; };
__global__ void __launch_bounds__(256) bloom_probe_kernel(const BloomProbeDev* __restrict__ probes, uint32_t n, const uint64_t* __restrict__ hashes,
                                                          uint8_t* __restrict__ maybe) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const BloomProbeDev q = probes[i];
  uint8_t m = 0;
  for (uint32_t j = 0; j < q.count && !m; j++) m = bloom::may_contain(q.bits, q.nblocks, hashes[q.first + j]) ? 1 : 0;
  maybe[i] = m;
}

// Bloom-filter pruning of the row groups that survived statistics, for resident files (their bitsets are in HBM inside the file
// bytes): one probe kernel and one small copy back, only when some surviving row group has a filter on an `=` / `IN` column.
int bloom_prune_resident(hg_engine* e, const hg_schema_desc* schema, const hg_predicate* preds, size_t np, std::vector<FileSel>& fs) {
  BloomLits bl;
  bloom_literals(schema, preds, np, &bl);
  if (!bl.n) return HG_OK;
  std::vector<BloomProbeDev> probes;
  std::vector<std::pair<uint32_t, uint32_t>> owner;        // (file, index into its rgs) of every probe
  for (size_t i = 0; i < fs.size(); i++) {
    const SstResident& f = *fs[i].f;
    const size_t ncols = size_t(f.meta.ncols);
    for (size_t x = 0; x < fs[i].rgs.size(); x++)
      for (size_t k = 0; k < bl.n; k++) {
        const RgCol& c = f.rgcol[size_t(fs[i].rgs[x]) * ncols + bl.col[k]];
        if (!c.bloom_blocks) continue;
        probes.push_back(BloomProbeDev{f.d_bytes + c.bloom_off, c.bloom_blocks, bl.first[k], bl.first[k + 1] - bl.first[k], 0});
        owner.emplace_back(uint32_t(i), uint32_t(x));
      }
  }
  if (probes.empty()) return HG_OK;
  const uint32_t n = uint32_t(probes.size());
  DevBuf d_probes, d_hashes, d_maybe;
  CU_TRY(d_probes.alloc(probes.size() * sizeof(BloomProbeDev), e->stream));
  CU_TRY(d_hashes.alloc(bl.h.size() * 8, e->stream));
  CU_TRY(d_maybe.alloc(n, e->stream));
  int rc = stage_upload(e, d_probes.p, probes.data(), probes.size() * sizeof(BloomProbeDev));
  if (!rc) rc = stage_upload(e, d_hashes.p, bl.h.data(), bl.h.size() * 8);
  if (rc) return rc;
  bloom_probe_kernel<<<(n + 255) / 256, 256, 0, e->stream>>>(d_probes.as<BloomProbeDev>(), n, d_hashes.as<uint64_t>(), d_maybe.as<uint8_t>());
  e->launches++;
  CU_TRY(cudaGetLastError());
  std::vector<uint8_t> maybe(n);
  CU_TRY(cudaMemcpyAsync(maybe.data(), d_maybe.p, n, cudaMemcpyDeviceToHost, e->stream));
  CU_TRY(cudaStreamSynchronize(e->stream));
  e->stats.bytes_h2d += probes.size() * sizeof(BloomProbeDev) + bl.h.size() * 8;
  e->stats.bytes_d2h += n;
  std::vector<std::vector<uint8_t>> drop(fs.size());
  for (size_t i = 0; i < fs.size(); i++) drop[i].assign(fs[i].rgs.size(), 0);
  for (uint32_t q = 0; q < n; q++) if (!maybe[q]) drop[owner[q].first][owner[q].second] = 1;
  for (size_t i = 0; i < fs.size(); i++) {
    size_t w = 0;
    for (size_t x = 0; x < fs[i].rgs.size(); x++) if (!drop[i][x]) fs[i].rgs[w++] = fs[i].rgs[x];
    fs[i].rgs.resize(w);
  }
  return HG_OK;
}
}  // namespace

// Row-group selection of a call, independent of the columns it reads: per file, the row groups that survive rg_dead, statistics and
// bloom pruning; then whether the inputs are provably PK-disjoint (plan->disjoint) and the decode order of the files (*sel, in it).
static int select_row_groups(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n, const hg_predicate* preds,
                             size_t np, std::vector<FileSel>* sel, ScanPlan* plan) {
  const bool prune = !(e->flags & HG_FLAG_NO_PRUNING);
  const auto tsel0 = HostClock::now();
  std::vector<FileSel> fs(n);
  uint64_t lits[MAX_PREDS];
  for (size_t i = 0; i < np; i++) lits[i] = pred_literal(preds[i], schema->types[preds[i].column]);
  for (size_t i = 0; i < n; i++) {
    auto it = e->ssts.find(ssts[i].id);
    if (it == e->ssts.end()) return set_error(HG_ERR_INTERNAL, "sst not resident after load");
    fs[i].f = it->second.get();
    const SstResident& f = *fs[i].f;
    const size_t nrg = f.rg_rows.size();
    fs[i].rgs.reserve(nrg);
    for (size_t g = 0; g < nrg; g++) {
      const uint32_t rows = f.rg_rows[g];
      plan->rows_in_files += rows;
      if (rows == 0) continue;
      if (!f.rg_dead.empty() && f.rg_dead[g]) continue;          // transient load: no row of this row group passes the predicate
      if (prune && np && !rg_may_match(f, g, schema, preds, lits, np, e->in_sets)) continue;
      fs[i].rgs.push_back(uint32_t(g));
    }
  }
  if (trace_on()) fprintf(stderr, "[plan] statistics pruning of %zu files: %.0f us\n", n, elapsed_us(tsel0, HostClock::now()));
  if (prune && np && !(e->flags & HG_FLAG_NO_BLOOM_FILTER)) {
    const int rc = bloom_prune_resident(e, schema, preds, np, fs);
    if (rc) return rc;
  }
  // PK-disjointness from the pk0 chunk statistics of the selected row groups of the files that keep any; those files lead the decode
  // order, by min(pk0), the others follow in the order given
  std::vector<size_t> order(n);
  for (size_t i = 0; i < n; i++) order[i] = i;
  plan->disjoint = n <= 1;
  if (n > 1) {
    std::vector<size_t> nonempty, by_pk0;
    std::vector<Pk0Range> ranges;
    for (size_t i = 0; i < n; i++) {
      if (fs[i].rgs.empty()) continue;
      nonempty.push_back(i);
      ranges.emplace_back();
      for (uint32_t g : fs[i].rgs) ranges.back().add(fs[i].f->rgcol[g * size_t(fs[i].f->meta.ncols)], schema->types[0]);
    }
    if (pk0_disjoint(ranges, schema->types[0], &by_pk0)) {
      plan->disjoint = true;
      order.clear();
      for (size_t x : by_pk0) order.push_back(nonempty[x]);
      for (size_t i = 0; i < n; i++) if (fs[i].rgs.empty()) order.push_back(i);
    }
  }
  sel->clear();
  for (size_t i : order) sel->push_back(std::move(fs[i]));
  return HG_OK;
}

// Layout of the selected row groups for the columns a call decodes: the RgSel table, scratch offsets, which columns may hold NULLs,
// the reader's batch boundaries (single file) and whether every chunk is one uncompressed PLAIN page.
static int lay_out_plan(const hg_engine* e, const hg_schema_desc* schema, const std::vector<FileSel>& fs, const std::vector<uint32_t>& need_cols,
                        ScanPlan* plan) {
  const size_t n = fs.size();
  size_t total_rgs = 0;
  for (const FileSel& f : fs) total_rgs += f.rgs.size();
  plan->col_has_nulls.assign(schema->num_columns, false);
  plan->sel.reserve(total_rgs);
  std::vector<uint8_t> has_nulls(schema->num_columns, 0);
  uint64_t row = 0, scratch = 0;
  for (size_t oi = 0; oi < n; oi++) {
    const FileSel& f = fs[oi];
    plan->files.push_back(f.f);
    plan->file_base.push_back(uint32_t(row));
    const size_t ncols = size_t(f.f->meta.ncols);
    for (uint32_t g : f.rgs) {
      const uint32_t rows = f.f->rg_rows[g];
      const RgCol* rc = &f.f->rgcol[size_t(g) * ncols];
      RgSel s;
      s.sst = uint32_t(oi);
      s.rg = g;
      s.out_row = uint32_t(row);
      s.num_rows = rows;
      s.scratch_off = scratch;
      for (uint32_t c : need_cols) {
        const RgCol& cc = rc[c];
        scratch += cc.scratch;             // 0 for uncompressed PLAIN chunks
        if (!cc.null_none) has_nulls[c] = 1;
      }
      plan->sel.push_back(s);
      if (n == 1) {
        for (uint64_t b = e->batch_size; b < rows; b += e->batch_size) plan->piece_end.push_back(uint32_t(row + b));
        plan->piece_end.push_back(uint32_t(row + rows));
      }
      row += rows;
      if (row >= 0xfffffff0ull) return set_error(HG_ERR_UNSUPPORTED, "more than 2^32 rows in one scan call");
    }
  }
  for (uint32_t c = 0; c < schema->num_columns; c++) plan->col_has_nulls[c] = has_nulls[c] != 0;
  plan->file_base.push_back(uint32_t(row));
  plan->rows_decoded = row;
  plan->scratch_bytes = scratch;
  return HG_OK;
}

// ------------------------------------------------------------------------------------------- the general pipeline
struct DecodedCol {
  DevBuf vals, valid, lens;            // lens: Binary columns only (vals = one byte pointer per row)
  uint32_t type = 0, width = 0;
  ColView view() const { return ColView{vals.p, reinterpret_cast<const uint8_t*>(valid.p), type, width, reinterpret_cast<const uint32_t*>(lens.p)}; }
};

struct PipelineState {
  ScanPlan plan;
  std::vector<DecodedCol> cols;       // indexed by schema column
  uint32_t N = 0;                     // decoded rows (capacity of every row-indexed buffer)
  DevBuf d_ssts, d_sel, d_colsel, d_scratch, d_err, d_counters;   // counters: [0]=M survivors [1]=R outputs [2]=G groups
  DevBuf d_dba_pages, d_dba_base, d_dba;   // DELTA_BYTE_ARRAY pages: descriptors, first descriptor per decode block, the values (rows point there)
  uint64_t d2h = 0;                        // device-to-host bytes of the pipeline itself (the DELTA_BYTE_ARRAY sizes)
  DevBuf alive, surv, keep, out_pos, out_rows, tmp, run_start, file_base, recA, recB, order, chunk_end, piece_end, bound;
  uint32_t nchunks = 0;
  const uint32_t* surv_ptr = nullptr;    // nullptr = identity
  bool keep_order = false;               // Append mode: the export needs the merged order of ALL surviving rows
  const uint32_t* order_ptr = nullptr;   //   row id of the t-th surviving row in merged order (nullptr = identity), valid when keep_order
  const uint32_t* d_m = nullptr;
  const uint32_t* d_r = nullptr;
  const uint32_t* d_g = nullptr;
  uint32_t* counters() const { return d_counters.as<uint32_t>(); }
};

static int validate_schema(const hg_schema_desc* s) {
  if (!s || !s->types) return set_error(HG_ERR_INVALID, "null schema");
  if (s->num_primary_keys == 0) return set_error(HG_ERR_INVALID, "num_primary_keys should large than 0");  // types.rs:165
  if (s->num_columns < s->num_primary_keys + 3 || s->num_columns > uint32_t(MAX_COLS))
    return set_error(HG_ERR_INVALID, "schema needs pk columns, at least one value column and the two builtin columns");
  if (s->num_primary_keys > uint32_t(MAX_PK)) return set_error(HG_ERR_UNSUPPORTED, "more than 4 primary key columns");
  if (s->update_mode > HG_UPDATE_APPEND) return set_error(HG_ERR_INVALID, "bad update mode");
  uint32_t pk_bytes = 0;
  for (uint32_t c = 0; c < s->num_columns; c++) if (s->types[c] > T_BINARY) return set_error(HG_ERR_INVALID, "bad column type");
  if (s->update_mode == HG_UPDATE_APPEND)       // read.rs:485-490 + operator.rs:66-73: BytesMergeOperator over ALL value columns
    for (uint32_t c = s->num_primary_keys; c + 2 < s->num_columns; c++)
      if (s->types[c] != T_BINARY) return set_error(HG_ERR_INVALID, "MergeOperator is only used for binary column (UpdateMode::Append)");
  for (uint32_t c = 0; c < s->num_primary_keys; c++) {
    uint32_t t = s->types[c];
    // primary_key_eq supports exactly these (read.rs:269-286); other types silently compare equal there — fenced off here
    if (!(t == T_U8 || t == T_I8 || t == T_U32 || t == T_I32 || t == T_U64 || t == T_I64))
      return set_error(HG_ERR_UNSUPPORTED, "primary key type not supported by the reference's primary_key_eq");
    pk_bytes += type_width(t);
  }
  if (pk_bytes > 16) return set_error(HG_ERR_UNSUPPORTED, "primary key wider than 128 bits");
  if (s->types[s->num_columns - 2] != T_U64 || s->types[s->num_columns - 1] != T_U64)
    return set_error(HG_ERR_INVALID, "builtin columns must be UInt64");
  return HG_OK;
}

static int validate_preds(const hg_schema_desc* s, const hg_predicate* preds, size_t np) {
  if (np > size_t(MAX_PREDS)) return set_error(HG_ERR_UNSUPPORTED, "more than 8 predicates");
  for (size_t i = 0; i < np; i++) {
    if (preds[i].column >= s->num_columns) return set_error(HG_ERR_INVALID, "predicate column out of range");
    if (preds[i].op > HG_OP_IN_SET) return set_error(HG_ERR_UNSUPPORTED, "predicate operator");
    if (preds[i].op == HG_OP_IN_SET) {
      const uint32_t t = s->types[preds[i].column];
      if (t == T_BINARY || type_is_float(t))
        return set_error(HG_ERR_UNSUPPORTED, std::string("IN_SET on column '") + (s->names && s->names[preds[i].column] ? s->names[preds[i].column] : "?") +
                                                 "': set predicates are implemented for integer columns only");
      if (preds[i].in_count > HG_MAX_IN_SET || (preds[i].in_count && !preds[i].in_values))
        return set_error(HG_ERR_INVALID, "IN_SET: null pointer or more than HG_MAX_IN_SET values");
      continue;
    }
    if (s->types[preds[i].column] == T_BINARY) {           // literals in in_bytes[0 .. in_count), for every operator
      const hg_predicate& p = preds[i];
      if (!p.in_bytes) return set_error(HG_ERR_INVALID, "Binary predicate: null in_bytes");
      if (p.op != HG_OP_IN && p.in_count != 1) return set_error(HG_ERR_INVALID, "Binary comparison: in_count must be 1");
      if (p.in_count > HG_MAX_IN_LIST) return set_error(HG_ERR_INVALID, "IN list: more than HG_MAX_IN_LIST values");
      for (uint32_t j = 0; j < p.in_count; j++) {
        if (p.in_bytes[j].len > HG_MAX_BINARY_LITERAL) return set_error(HG_ERR_INVALID, "Binary literal larger than HG_MAX_BINARY_LITERAL bytes");
        if (!p.in_bytes[j].data && p.in_bytes[j].len) return set_error(HG_ERR_INVALID, "Binary literal: null data with a non-zero length");
      }
      continue;
    }
    if (preds[i].op == HG_OP_IN && (preds[i].in_count > HG_MAX_IN_LIST || (preds[i].in_count && !preds[i].in_values)))
      return set_error(HG_ERR_INVALID, "IN list: null pointer or more than HG_MAX_IN_LIST values");
  }
  return HG_OK;
}

// --- S2: decode the needed columns of the selected row groups, DELTA_BYTE_ARRAY values included
static int decode_stage(hg_engine* e, const hg_schema_desc* schema, const std::vector<uint32_t>& need_cols, PipelineState* st) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const auto tp0 = HostClock::now();
  const ScanPlan& plan = st->plan;
  const uint32_t N = st->N;
  st->cols.resize(schema->num_columns);
  std::vector<ColSel> colsel;
  for (uint32_t c : need_cols) {
    DecodedCol& dc = st->cols[c];
    dc.type = schema->types[c];
    dc.width = type_width(dc.type);
    CU_TRY(dc.vals.alloc(size_t(N) * dc.width + 16, s));
    if (plan.col_has_nulls[c] || dc.type == T_BINARY) CU_TRY(dc.valid.alloc(size_t(N) + 16, s));
    if (dc.type == T_BINARY) CU_TRY(dc.lens.alloc(size_t(N) * 4 + 16, s));
    ColSel cs;
    cs.col = c;
    cs.type = dc.type;
    cs.out_width = dc.width;
    cs._pad = 0;
    cs.out_vals = dc.vals.p;
    cs.out_valid = reinterpret_cast<uint8_t*>(dc.valid.p);
    cs.out_lens = reinterpret_cast<uint32_t*>(dc.lens.p);
    colsel.push_back(cs);
  }
  if (N > 0) {
    std::vector<SstDev> sd(plan.files.size());
    for (size_t i = 0; i < plan.files.size(); i++) {
      SstResident* f = plan.files[i];
      sd[i] = SstDev{f->d_bytes, f->d_pages, f->d_chunks, uint32_t(f->meta.ncols), uint32_t(f->meta.rgs.size())};
    }
    CU_TRY(st->d_ssts.alloc(sd.size() * sizeof(SstDev), s));
    CU_TRY(st->d_sel.alloc(plan.sel.size() * sizeof(RgSel), s));
    CU_TRY(st->d_colsel.alloc(colsel.size() * sizeof(ColSel), s));
    int urc = stage_upload(e, st->d_ssts.p, sd.data(), sd.size() * sizeof(SstDev));
    if (!urc) urc = stage_upload(e, st->d_sel.p, plan.sel.data(), plan.sel.size() * sizeof(RgSel));
    if (!urc) urc = stage_upload(e, st->d_colsel.p, colsel.data(), colsel.size() * sizeof(ColSel));
    if (urc) return urc;
    // DELTA_BYTE_ARRAY pages of the selected Binary chunks: decode_chunks sizes each into a descriptor, numbered in (row group, column,
    // page) order.  Calls without such pages allocate, copy and launch nothing for them.
    bool any_binary = false;
    for (const ColSel& c : colsel) any_binary = any_binary || c.type == T_BINARY;
    uint32_t ndba = 0;
    std::vector<uint32_t> dba_base;                          // per decode block (row group si, column ci): DELTA_BYTE_ARRAY pages before it
    if (any_binary) {
      dba_base.resize(plan.sel.size() * colsel.size());
      for (size_t si = 0; si < plan.sel.size(); si++) {
        const FileMetaData& m = plan.files[plan.sel[si].sst]->meta;
        for (size_t ci = 0; ci < colsel.size(); ci++) {
          dba_base[si * colsel.size() + ci] = ndba;
          if (colsel[ci].type != T_BINARY) continue;
          const ChunkMeta& cm = m.rgs[plan.sel[si].rg].cols[colsel[ci].col];
          for (uint32_t pi = cm.first_page; pi < cm.first_page + cm.num_pages; pi++) ndba += m.pages[pi].encoding == ENC_DELTA_BYTE_ARRAY ? 1u : 0u;
        }
      }
    }
    if (ndba) {
      CU_TRY(st->d_dba_pages.alloc(size_t(ndba) * sizeof(DbaPage), s));
      CU_TRY(st->d_dba_base.alloc(dba_base.size() * sizeof(uint32_t), s));
      CU_TRY(cudaMemsetAsync(st->d_dba_pages.p, 0, size_t(ndba) * sizeof(DbaPage), s));
      urc = stage_upload(e, st->d_dba_base.p, dba_base.data(), dba_base.size() * sizeof(uint32_t));
      if (urc) return urc;
    }
    // the host vectors must outlive the async copies: pageable memcpy is staged synchronously by the runtime
    const auto tp1 = HostClock::now();
    CU_TRY(cudaEventRecord(e->evk0, s));
    if (plan.scratch_bytes) {
      CU_TRY(st->d_scratch.alloc(plan.scratch_bytes + 64, s));
      k::snappy_chunks(L, st->d_ssts.as<SstDev>(), st->d_sel.as<RgSel>(), uint32_t(plan.sel.size()), st->d_colsel.as<ColSel>(),
                       int(colsel.size()), st->d_scratch.as<uint8_t>(), st->counters() + 4, st->d_err.as<int>());
      bool any_zstd = false;
      for (const SstResident* f : plan.files) any_zstd = any_zstd || f->any_zstd;
      if (any_zstd)                                          // ParquetCompression::Zstd (config.rs:78-94): its own kernel, same scratch layout
        k::zstd_chunks(L, st->d_ssts.as<SstDev>(), st->d_sel.as<RgSel>(), uint32_t(plan.sel.size()), st->d_colsel.as<ColSel>(),
                       int(colsel.size()), st->d_scratch.as<uint8_t>(), st->counters() + 6, st->d_err.as<int>());
    }
    k::decode_chunks(L, st->d_ssts.as<SstDev>(), st->d_sel.as<RgSel>(), uint32_t(plan.sel.size()), st->d_colsel.as<ColSel>(),
                     int(colsel.size()), st->d_scratch.as<uint8_t>(), st->d_dba_pages.as<DbaPage>(), st->d_dba_base.as<uint32_t>(),
                     st->d_err.as<int>());
    if (ndba) {
      // DELTA_BYTE_ARRAY: the page sizes come back (one small copy, one synchronisation), an exclusive scan places every page in one
      // buffer that lives as long as the scratch, and one warp per page writes the values.  A page that failed validation has size 0
      // and keeps its rows NULL; the call reports HG_ERR_FORMAT from the error word.
      std::vector<DbaPage> hp(ndba);
      CU_TRY(cudaMemcpyAsync(hp.data(), st->d_dba_pages.p, size_t(ndba) * sizeof(DbaPage), cudaMemcpyDeviceToHost, s));
      CU_TRY(cudaStreamSynchronize(s));
      st->d2h += uint64_t(ndba) * sizeof(DbaPage);
      uint64_t total = 0;
      for (DbaPage& d : hp) { d.out_off = total; total += d.bytes; }
      if (total >= 0x7fffffffu) return set_error(HG_ERR_UNSUPPORTED, "DELTA_BYTE_ARRAY values larger than 2 GiB in one call (Arrow int32 offsets)");
      CU_TRY(st->d_dba.alloc(size_t(total) + 64, s));
      urc = stage_upload(e, st->d_dba_pages.p, hp.data(), size_t(ndba) * sizeof(DbaPage));
      if (urc) return urc;
      k::dba_materialise(L, st->d_dba_pages.as<DbaPage>(), ndba, st->d_colsel.as<ColSel>(), st->d_dba.as<uint8_t>());
    }
    CU_TRY(cudaEventRecord(e->evk1, s));
    bool rows_point_into_scratch = false;                   // Binary rows are pointers to their bytes in place (page or decompression scratch)
    for (uint32_t c : need_cols) if (schema->types[c] == T_BINARY) rows_point_into_scratch = true;
    if (!rows_point_into_scratch) st->d_scratch.reset();
    if (trace_on())
      fprintf(stderr, "[general] col alloc+upload %.0f us, scratch alloc (%.1f MB) + decode launches %.0f us\n", elapsed_us(tp0, tp1), plan.scratch_bytes / 1e6,
              elapsed_us(tp1, HostClock::now()));
  }
  return HG_OK;
}

// The literals of a call's predicates on the device: the IN lists of fixed-width columns one by one, the Binary literals as one blob
// (their BinLitDev table, then their bytes) in one upload
static int stage_predicates(hg_engine* e, const hg_schema_desc* schema, const hg_predicate* preds, size_t np, const PipelineState* st,
                            PredSet* ps, BinPredSet* bs, InSetPreds* is) {
  ps->n = 0;
  bs->n = 0;
  bs->n_lits = 0;
  bs->lits = nullptr;
  is->n = 0;
  for (size_t i = 0; i < np; i++) {
    if (preds[i].op == HG_OP_IN_SET) {
      // The sorted keys go up once, straight from the call's host copy (it outlives the call's device work): a set can be far larger
      // than the staging buffer is meant to become
      const std::vector<uint64_t>& keys = e->in_sets.keys[i];
      uint64_t* d_keys = static_cast<uint64_t*>(g_arena->alloc(std::max<size_t>(keys.size(), 1) * 8));
      if (!d_keys) return set_error(HG_ERR_OOM, "out of device memory");
      if (!keys.empty()) CU_TRY(cudaMemcpyAsync(d_keys, keys.data(), keys.size() * 8, cudaMemcpyHostToDevice, e->stream));
      e->stats.bytes_h2d += keys.size() * 8;
      e->in_sets.dev[i] = d_keys;
      is->p[is->n++] = InSetDev{st->cols[preds[i].column].view(), d_keys, uint32_t(keys.size()), 0};
      continue;
    }
    if (schema->types[preds[i].column] == T_BINARY) {
      BinPredDev& b = bs->p[bs->n++];
      b.col = st->cols[preds[i].column].view();
      b.op = preds[i].op;
      b.first = bs->n_lits;
      b.n_lit = preds[i].in_count;               // 1 for a comparison (validate_preds)
      b._pad = 0;
      bs->n_lits += preds[i].in_count;
      continue;
    }
    PredDev& pd = ps->p[ps->n++];
    pd.col = st->cols[preds[i].column].view();
    pd.op = preds[i].op;
    pd.n_in = 0;
    pd.in_list = nullptr;
    pd.lit = pred_literal(preds[i], schema->types[preds[i].column]);
    if (preds[i].op == HG_OP_IN) {
      uint64_t* d_list = static_cast<uint64_t*>(g_arena->alloc(std::max<size_t>(preds[i].in_count, 1) * 8));
      if (!d_list) return set_error(HG_ERR_OOM, "out of device memory");
      if (preds[i].in_count) {
        int urc = stage_upload(e, d_list, preds[i].in_values, size_t(preds[i].in_count) * 8);
        if (urc) return urc;
      }
      pd.n_in = preds[i].in_count;
      pd.in_list = d_list;
    }
  }
  if (bs->n) {
    size_t bytes = size_t(bs->n_lits) * sizeof(BinLitDev);
    for (size_t i = 0; i < np; i++)
      if (schema->types[preds[i].column] == T_BINARY)
        for (uint32_t j = 0; j < preds[i].in_count; j++) bytes += preds[i].in_bytes[j].len;
    uint8_t* d_blob = static_cast<uint8_t*>(g_arena->alloc(std::max<size_t>(bytes, 16)));   // no slack: a compare reads no byte past a literal
    if (!d_blob) return set_error(HG_ERR_OOM, "out of device memory");
    std::vector<uint8_t> blob(bytes);
    size_t off = size_t(bs->n_lits) * sizeof(BinLitDev), t = 0;
    for (size_t i = 0; i < np; i++) {
      if (schema->types[preds[i].column] != T_BINARY) continue;
      for (uint32_t j = 0; j < preds[i].in_count; j++, t++) {
        const hg_bytes& lb = preds[i].in_bytes[j];
        if (lb.len) std::memcpy(blob.data() + off, lb.data, lb.len);
        const BinLitDev l{bytes_key(blob.data() + off, lb.len), d_blob + off, uint32_t(lb.len), 0};
        std::memcpy(blob.data() + t * sizeof(BinLitDev), &l, sizeof(l));
        off += lb.len;
      }
    }
    if (bytes) {
      int urc = stage_upload(e, d_blob, blob.data(), blob.size());
      if (urc) return urc;
    }
    bs->lits = reinterpret_cast<const BinLitDev*>(d_blob);
  }
  return HG_OK;
}

// --- S3: filter (before the merge, read.rs:459-470)
static int filter_stage(hg_engine* e, const hg_schema_desc* schema, const hg_predicate* preds, size_t np, PipelineState* st) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const uint32_t N = st->N;
  CU_TRY(st->tmp.alloc(k::compact_tmp_elems(N) * sizeof(uint32_t), s));
  if (np > 0 && N > 0) {
    PredSet ps;
    BinPredSet bs;
    InSetPreds is;
    int rc = stage_predicates(e, schema, preds, np, st, &ps, &bs, &is);
    if (rc) return rc;
    CU_TRY(st->alive.alloc(size_t(N) + 16, s));
    CU_TRY(st->surv.alloc(size_t(N) * 4 + 16, s));
    if (ps.n || (!bs.n && !is.n)) k::eval_predicates(L, ps, N, st->alive.as<uint8_t>());
    if (bs.n) k::eval_binary_predicates(L, bs, N, ps.n > 0, st->alive.as<uint8_t>());
    if (is.n) k::eval_in_set(L, is, N, ps.n > 0 || bs.n > 0, st->alive.as<uint8_t>());
    k::compact_flags(L, st->alive.as<uint8_t>(), N, st->tmp.as<uint32_t>(), st->surv.as<uint32_t>(), st->counters() + 0);
    st->alive.reset();
    st->surv_ptr = st->surv.as<uint32_t>();
  } else {
    k::fill_u32(L, st->counters() + 0, N, 1);
    st->surv_ptr = nullptr;
  }
  return HG_OK;
}

// Packing of the merge key (pk..., __seq__, stream) into one 64-bit word, each field rebased to the statistics of the selected chunks.
// False when some chunk has no statistics or the fields need more than 52 bits.
static bool plan_key_pack(const ScanPlan& plan, const hg_schema_desc* schema, int k, k::KeyPack* kp) {
  std::memset(kp, 0, sizeof(*kp));
  const int npk = int(schema->num_primary_keys);
  const uint32_t seq_idx = schema->num_columns - 2;
  uint64_t lo[MAX_PK + 1], hi[MAX_PK + 1];
  bool seen_c[MAX_PK + 1] = {false};
  bool seq_nullable = false;
  for (int c = 0; c <= MAX_PK; c++) { lo[c] = 0; hi[c] = 0; }
  if (plan.sel.empty()) return false;
  for (const RgSel& rs : plan.sel) {
    const SstResident* f = plan.files[rs.sst];
    const RgCol* rc = &f->rgcol[size_t(rs.rg) * size_t(f->meta.ncols)];
    for (int c = 0; c <= npk; c++) {
      const uint32_t col = c < npk ? uint32_t(c) : seq_idx;
      const RgCol& x = rc[col];
      if (c == npk && x.null_all) { seq_nullable = true; continue; }
      if (!x.has_minmax) return false;
      const uint64_t flip = c < npk ? order_flip(schema->types[col]) : 0ull;
      const uint64_t a = x.mn ^ flip, b = x.mx ^ flip;
      if (c == npk && !x.null_none) seq_nullable = true;
      if (!seen_c[c] || a < lo[c]) lo[c] = a;
      if (!seen_c[c] || b > hi[c]) hi[c] = b;
      seen_c[c] = true;
    }
  }
  if (!seen_c[npk]) { seq_nullable = true; lo[npk] = 0; hi[npk] = 0; }      // every __seq__ chunk is all-null
  auto bits = [](uint64_t span) { int b = 0; while (span) { b++; span >>= 1; } return b; };
  int rb = 0;
  while ((1 << rb) < k) rb++;
  // seq lives in the (value + 1, NULL = 0) domain
  if (hi[npk] == ~0ull) return false;
  kp->seq_min = seq_nullable ? 0 : lo[npk] + 1;
  kp->seq_span = seen_c[npk] ? hi[npk] + 1 - kp->seq_min : 0;
  kp->seq_shift = uint32_t(rb);
  int used = rb + bits(kp->seq_span);
  kp->pk_shift = uint32_t(used);
  for (int c = npk - 1; c >= 0; c--) {
    kp->mn[c] = lo[c];
    kp->span[c] = hi[c] - lo[c];
    kp->shift[c] = uint32_t(used);
    used += bits(kp->span[c]);
  }
  return used <= 52;
}

// --- S4: merge on (pk..., __seq__) when the inputs are not provably PK-disjoint.  st->order_ptr: the surviving rows in merged order
static int merge_stage(hg_engine* e, const hg_schema_desc* schema, PipelineState* st) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const ScanPlan& plan = st->plan;
  const uint32_t N = st->N;
  const int k = int(plan.files.size());
  const uint32_t seq_idx = schema->num_columns - 2;
  PkSet pk;
  pk.n = int(schema->num_primary_keys);
  for (int c = 0; c < pk.n; c++) {
    pk.c[c] = st->cols[c].view();
    if (plan.col_has_nulls[c]) return set_error(HG_ERR_UNSUPPORTED, "NULL primary keys are not supported on the GPU path");
  }
  const uint32_t* order = st->surv_ptr;
  CU_TRY(st->keep.alloc(size_t(N) + 16, s));
  CU_TRY(cudaEventRecord(e->evm0, s));
  if (!plan.disjoint && N > 0) {
    CU_TRY(st->file_base.alloc((k + 1) * sizeof(uint32_t), s));
    CU_TRY(st->run_start.alloc((k + 2) * sizeof(uint32_t), s));
    CU_TRY(cudaMemcpyAsync(st->file_base.p, plan.file_base.data(), (k + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    k::survivor_run_starts(L, st->surv_ptr, st->d_m, st->file_base.as<uint32_t>(), k, st->run_start.as<uint32_t>());
    // single pass over packed 64-bit keys when (pk..., __seq__, stream) fit in 52 bits after rebasing to the chunk statistics
    k::KeyPack kp;
    const bool packed = k <= k::kMaxMergeRuns && !(e->flags & HG_FLAG_PAIRWISE_MERGE) && plan_key_pack(plan, schema, k, &kp);
    if (packed) {
      uint32_t ranges = 1;
      DevBuf ktmp;
      CU_TRY(ktmp.alloc(k::kway_tmp_bytes(N, k, &ranges), s));
      CU_TRY(st->order.alloc(size_t(N) * 4 + 16, s));
      k::kway_merge(L, pk, st->cols[seq_idx].view(), st->surv_ptr, st->d_m, N, st->run_start.as<uint32_t>(), k, kp, ktmp.p,
                    st->counters() + 5, st->order.as<uint32_t>(), st->keep.as<uint8_t>(), st->d_err.as<int>());
      order = st->order.as<uint32_t>();
      st->surv_ptr = nullptr;
    } else {
    CU_TRY(st->recA.alloc(size_t(N) * sizeof(SortRec) + 32, s));
    CU_TRY(st->recB.alloc(size_t(N) * sizeof(SortRec) + 32, s));
    k::build_records(L, pk, st->cols[seq_idx].view(), st->surv_ptr, st->d_m, N, st->recA.as<SortRec>());
    DevBuf splits;
    CU_TRY(splits.alloc(k::merge_split_elems(N) * sizeof(uint32_t), s));
    SortRec* src = st->recA.as<SortRec>();
    SortRec* dst = st->recB.as<SortRec>();
    for (int level = 0; (1 << level) < k; level++) {
      k::merge_pass(L, src, dst, st->run_start.as<uint32_t>(), k, level, st->d_m, N, splits.as<uint32_t>());
      std::swap(src, dst);
    }
    CU_TRY(st->order.alloc(size_t(N) * 4 + 16, s));
    k::records_to_rows(L, src, st->d_m, N, st->order.as<uint32_t>());
    k::dedup_flags_recs(L, src, st->d_m, N, st->keep.as<uint8_t>());
    order = st->order.as<uint32_t>();
    st->recA.reset();
    st->recB.reset();
    st->surv_ptr = nullptr;  // (no longer valid)
    }
    st->surv.reset();
  } else if (N > 0) {
    k::dedup_flags_cols(L, pk, order, st->d_m, N, st->keep.as<uint8_t>());
  }
  st->order_ptr = order;
  return HG_OK;
}

// --- S5/S6: keep the last row of every PK run, and the batch boundaries of MergeStream
static int dedup_stage(hg_engine* e, bool want_batches, PipelineState* st) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const uint32_t N = st->N;
  const int k = int(st->plan.files.size());
  const uint32_t* order = st->order_ptr;
  // batch boundaries of MergeStream need the chunking of its INPUT (computed before surv is dropped)
  if (want_batches && N > 0) {
    if (k == 1) {
      st->nchunks = uint32_t(st->plan.piece_end.size());
      CU_TRY(st->piece_end.alloc(st->nchunks * sizeof(uint32_t) + 16, s));
      CU_TRY(st->chunk_end.alloc(st->nchunks * sizeof(uint32_t) + 16, s));
      CU_TRY(cudaMemcpyAsync(st->piece_end.p, st->plan.piece_end.data(), st->nchunks * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
      k::chunk_ends_from_rows(L, order /* == surv or identity */, st->d_m, st->piece_end.as<uint32_t>(), st->nchunks,
                              st->chunk_end.as<uint32_t>());
    } else {
      st->nchunks = (N + e->batch_size - 1) / e->batch_size;
      CU_TRY(st->chunk_end.alloc(st->nchunks * sizeof(uint32_t) + 16, s));
      k::uniform_chunk_ends(L, st->d_m, e->batch_size, st->nchunks, st->chunk_end.as<uint32_t>());
    }
  }
  CU_TRY(st->out_pos.alloc(size_t(N) * 4 + 16, s));
  CU_TRY(st->out_rows.alloc(size_t(N) * 4 + 16, s));
  if (N > 0) {
    // compaction over the first M flags only: flags beyond M are stale, so clear the tail by bounding n on device
    k::clear_tail(L, st->keep.as<uint8_t>(), st->d_m, N);
    k::compact_flags(L, st->keep.as<uint8_t>(), N, st->tmp.as<uint32_t>(), st->out_pos.as<uint32_t>(), st->counters() + 1);
    k::gather_rows(L, order, st->out_pos.as<uint32_t>(), st->d_r, N, st->out_rows.as<uint32_t>());
    if (want_batches && st->nchunks) {
      CU_TRY(st->bound.alloc(st->nchunks * sizeof(uint32_t) + 16, s));
      k::batch_bounds(L, st->out_pos.as<uint32_t>(), st->d_r, st->chunk_end.as<uint32_t>(), st->nchunks, st->bound.as<uint32_t>());
    }
  }
  CU_TRY(cudaEventRecord(e->evm1, s));
  st->keep.reset();
  if (st->keep_order) return HG_OK;                  // (order_ptr points into st->order or st->surv: both stay allocated)
  st->order.reset();
  st->surv.reset();
  st->order_ptr = nullptr;
  return HG_OK;
}

// Runs decode -> filter -> merge -> dedup.  On return st->out_rows holds the surviving row ids in stream order,
// counters()[0..1] = M, R (device), st->out_pos their merged positions.
static int run_pipeline(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n, const hg_predicate* preds,
                        size_t np, std::vector<uint32_t> need_cols, bool want_batches, PipelineState* st) {
  // PKs are always needed (dedup); __seq__ whenever a real merge happens, i.e. the inputs are not provably PK-disjoint
  for (uint32_t c = 0; c < schema->num_primary_keys; c++) need_cols.push_back(c);
  for (size_t i = 0; i < np; i++) need_cols.push_back(preds[i].column);
  std::vector<FileSel> sel;
  int rc = select_row_groups(e, schema, ssts, n, preds, np, &sel, &st->plan);
  if (rc) return rc;
  if (!st->plan.disjoint) need_cols.push_back(schema->num_columns - 2);
  std::sort(need_cols.begin(), need_cols.end());
  need_cols.erase(std::unique(need_cols.begin(), need_cols.end()), need_cols.end());
  rc = lay_out_plan(e, schema, sel, need_cols, &st->plan);
  if (rc) return rc;
  st->N = uint32_t(st->plan.rows_decoded);

  cudaStream_t s = e->stream;
  CU_TRY(st->d_counters.alloc(8 * sizeof(uint32_t), s));
  CU_TRY(cudaMemsetAsync(st->d_counters.p, 0, 8 * sizeof(uint32_t), s));
  CU_TRY(st->d_err.alloc(sizeof(int), s));
  CU_TRY(cudaMemsetAsync(st->d_err.p, 0, sizeof(int), s));
  st->d_m = st->counters() + 0;
  st->d_r = st->counters() + 1;
  st->d_g = st->counters() + 2;

  rc = decode_stage(e, schema, need_cols, st);
  if (!rc) rc = filter_stage(e, schema, preds, np, st);
  if (!rc) rc = merge_stage(e, schema, st);
  if (!rc) rc = dedup_stage(e, want_batches, st);
  return rc;
}

static int check_device_error(hg_engine* e, PipelineState* st) {
  int herr = 0;
  CU_TRY(cudaMemcpyAsync(&herr, st->d_err.p, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  CU_TRY(cudaStreamSynchronize(e->stream));
  if (herr == 130) return set_error(HG_ERR_INVALID, "failed to construct RecordBatch in BytesMergeOperator (a run of several rows whose Binary values are all empty)");
  if (herr == k::kErrGroupMapMiss) return set_error(HG_ERR_INTERNAL, "a row that passed the group map's set has no group");
  if (herr) return set_error(HG_ERR_FORMAT, "device decode error code " + std::to_string(herr));
  return HG_OK;
}

// The statistics of a finished general pipeline (synchronises); hc = its counters (M, R, G, ...)
static int pipeline_stats(hg_engine* e, PipelineState* st, uint32_t hc[8]) {
  CU_TRY(cudaMemcpyAsync(hc, st->d_counters.p, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
  int rc = check_device_error(e, st);
  if (rc) return rc;
  e->stats.rows_in_files = st->plan.rows_in_files;
  e->stats.rows_decoded = st->plan.rows_decoded;
  e->stats.rows_materialized = st->plan.rows_decoded;
  e->stats.rows_filtered = hc[0];
  e->stats.rows_out = hc[1];
  float ms = 0;
  if (st->N > 0) { cudaEventElapsedTime(&ms, e->evk0, e->evk1); e->stats.kernel_ms = ms; cudaEventElapsedTime(&ms, e->evm0, e->evm1); e->stats.merge_ms = ms; }
  return HG_OK;
}

// ----------------------------------------------------------------------------------------------- pinned host pool
// Result batches live in pinned host memory owned by the Arrow stream; cudaMallocHost is slow and synchronising, so
// released buffers go back to a process-wide free list (bounded) instead of being freed.
namespace {
struct PinnedPool {
  std::mutex mu;
  std::vector<std::pair<size_t, void*>> free_list;
  size_t pooled = 0;
  static constexpr size_t kMaxPooled = size_t(16) << 30;
  void* alloc(size_t bytes) {
    bytes = (bytes + 4095) & ~size_t(4095);
    {
      std::lock_guard<std::mutex> g(mu);
      size_t best = free_list.size();
      for (size_t i = 0; i < free_list.size(); i++)
        if (free_list[i].first >= bytes && free_list[i].first <= bytes * 2 + (1 << 20) && (best == free_list.size() || free_list[i].first < free_list[best].first)) best = i;
      if (best != free_list.size()) {
        void* p = free_list[best].second;
        pooled -= free_list[best].first;
        sizes[p] = free_list[best].first;
        free_list.erase(free_list.begin() + best);
        return p;
      }
    }
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
    std::lock_guard<std::mutex> g(mu);
    sizes[p] = bytes;
    return p;
  }
  void release(void* p) {
    if (!p) return;
    std::lock_guard<std::mutex> g(mu);
    auto it = sizes.find(p);
    size_t b = it == sizes.end() ? 0 : it->second;
    if (it != sizes.end()) sizes.erase(it);
    if (b && pooled + b <= kMaxPooled) { free_list.emplace_back(b, p); pooled += b; }
    else cudaFreeHost(p);
  }
  std::unordered_map<void*, size_t> sizes;
};
PinnedPool& pinned_pool() { static PinnedPool* p = new PinnedPool(); return *p; }
}  // namespace

// --------------------------------------------------------------------------------------------- Arrow C stream export
struct HostColumn {
  std::string name;
  uint32_t type = 0, width = 0;
  void* vals = nullptr;          // pinned host: the values — for Binary columns the concatenated bytes
  uint8_t* bitmap = nullptr;     // pinned host, nullptr = no nulls
  int32_t* offsets = nullptr;    // pinned host, Binary columns only: Arrow offsets (rows + 1)
  int64_t null_count = 0;
};
struct StreamData {
  std::vector<HostColumn> cols;
  std::vector<uint32_t> batch_start;  // nb+1 row offsets
  size_t next = 0;
  std::string last_error;
  ~StreamData() {
    for (auto& c : cols) {
      pinned_pool().release(c.vals);
      pinned_pool().release(c.bitmap);
      pinned_pool().release(c.offsets);
    }
  }
};
struct StreamPriv { std::shared_ptr<StreamData> data; };

static void schema_release(struct ArrowSchema* s) {
  if (!s || !s->release) return;
  for (int64_t i = 0; i < s->n_children; i++) {
    if (s->children[i]->release) s->children[i]->release(s->children[i]);
    delete s->children[i];
  }
  delete[] s->children;
  delete reinterpret_cast<std::string*>(s->private_data);
  s->release = nullptr;
}
static void fill_schema(struct ArrowSchema* out, const std::shared_ptr<StreamData>& d) {
  std::memset(out, 0, sizeof(*out));
  out->format = "+s";
  out->name = "";
  out->n_children = int64_t(d->cols.size());
  out->children = new ArrowSchema*[d->cols.size() ? d->cols.size() : 1];
  for (size_t i = 0; i < d->cols.size(); i++) {
    ArrowSchema* c = new ArrowSchema();
    std::memset(c, 0, sizeof(*c));
    std::string* nm = new std::string(d->cols[i].name);
    c->format = arrow_format(d->cols[i].type);
    c->name = nm->c_str();
    c->flags = ARROW_FLAG_NULLABLE;
    c->private_data = nm;
    c->release = [](struct ArrowSchema* s) { delete reinterpret_cast<std::string*>(s->private_data); s->release = nullptr; };
    out->children[i] = c;
  }
  out->private_data = nullptr;
  out->release = schema_release;
}
struct ArrayPriv { std::shared_ptr<StreamData> keep; const void* bufs[3]; };
static void child_release(struct ArrowArray* a) {
  if (!a || !a->release) return;
  delete reinterpret_cast<ArrayPriv*>(a->private_data);
  a->release = nullptr;
}
static void batch_release(struct ArrowArray* a) {
  if (!a || !a->release) return;
  for (int64_t i = 0; i < a->n_children; i++) {
    if (a->children[i]->release) a->children[i]->release(a->children[i]);
    delete a->children[i];
  }
  delete[] a->children;
  delete reinterpret_cast<ArrayPriv*>(a->private_data);
  a->release = nullptr;
}
static int stream_get_schema(struct ArrowArrayStream* st, struct ArrowSchema* out) {
  fill_schema(out, reinterpret_cast<StreamPriv*>(st->private_data)->data);
  return 0;
}
static int stream_get_next(struct ArrowArrayStream* st, struct ArrowArray* out) {
  auto d = reinterpret_cast<StreamPriv*>(st->private_data)->data;
  std::memset(out, 0, sizeof(*out));
  if (d->next + 1 >= d->batch_start.size()) { out->release = nullptr; return 0; }  // end of stream
  uint32_t lo = d->batch_start[d->next], hi = d->batch_start[d->next + 1];
  d->next++;
  ArrayPriv* top = new ArrayPriv{d, {nullptr, nullptr, nullptr}};
  out->length = hi - lo;
  out->null_count = 0;
  out->offset = 0;
  out->n_buffers = 1;
  out->buffers = top->bufs;
  out->n_children = int64_t(d->cols.size());
  out->children = new ArrowArray*[d->cols.size() ? d->cols.size() : 1];
  for (size_t i = 0; i < d->cols.size(); i++) {
    ArrowArray* c = new ArrowArray();
    std::memset(c, 0, sizeof(*c));
    const bool bin = d->cols[i].type == T_BINARY;          // Binary: validity, int32 offsets, data
    ArrayPriv* p = bin ? new ArrayPriv{d, {d->cols[i].bitmap, d->cols[i].offsets, d->cols[i].vals}}
                       : new ArrayPriv{d, {d->cols[i].bitmap, d->cols[i].vals, nullptr}};
    c->length = hi - lo;
    c->offset = lo;
    c->null_count = d->cols[i].bitmap ? -1 : 0;
    c->n_buffers = bin ? 3 : 2;
    c->buffers = p->bufs;
    c->private_data = p;
    c->release = child_release;
    out->children[i] = c;
  }
  out->private_data = top;
  out->release = batch_release;
  return 0;
}
static const char* stream_last_error(struct ArrowArrayStream* st) {
  auto d = reinterpret_cast<StreamPriv*>(st->private_data)->data;
  return d->last_error.empty() ? nullptr : d->last_error.c_str();
}
static void stream_release(struct ArrowArrayStream* st) {
  if (!st || !st->release) return;
  delete reinterpret_cast<StreamPriv*>(st->private_data);
  st->release = nullptr;
}
static void make_stream(struct ArrowArrayStream* out, std::shared_ptr<StreamData> d) {
  out->get_schema = stream_get_schema;
  out->get_next = stream_get_next;
  out->get_last_error = stream_last_error;
  out->release = stream_release;
  out->private_data = new StreamPriv{std::move(d)};
}

// ------------------------------------------------------------------------------------------------------------ C ABI
extern "C" {

uint32_t hg_abi_version(void) { return HG_ABI_VERSION; }
const char* hg_last_error(void) { return g_last_error.c_str(); }

int hg_engine_create(const hg_config* cfg, hg_engine** out) {
  HG_GUARD_BEGIN
  if (!cfg || !out) return set_error(HG_ERR_INVALID, "null argument");
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return set_error(HG_ERR_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(ce) + " (this library has no CPU fallback)");
  if (cfg->device < 0 || cfg->device >= ndev) return set_error(HG_ERR_INVALID, "device ordinal out of range");
  CU_TRY(cudaSetDevice(cfg->device));
  auto e = std::make_unique<hg_engine>();
  e->device = cfg->device;
  e->batch_size = cfg->batch_size ? cfg->batch_size : 8192;
  e->flags = cfg->flags;
  e->budget = cfg->hbm_budget_bytes;
  CU_TRY(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
  CU_TRY(cudaEventCreate(&e->ev0));
  CU_TRY(cudaEventCreate(&e->ev1));
  CU_TRY(cudaEventCreate(&e->evk0));
  CU_TRY(cudaEventCreate(&e->evk1));
  CU_TRY(cudaEventCreate(&e->evm0));
  CU_TRY(cudaEventCreate(&e->evm1));
  CU_TRY(cudaEventCreate(&e->evd0));
  CU_TRY(cudaEventCreate(&e->evd1));
  cudaMemPool_t pool;
  CU_TRY(cudaDeviceGetDefaultMemPool(&pool, cfg->device));
  uint64_t thresh = UINT64_MAX;
  CU_TRY(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
  *out = e.release();
  return HG_OK;
  HG_GUARD_END
}

void hg_engine_destroy(hg_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->stream);
  hg_comm_free(e->comm);
  e->comm = nullptr;
  g_arena = nullptr;
  e->arena.destroy();
  if (e->h_stage) cudaFreeHost(e->h_stage);
  if (e->h_small) cudaFreeHost(e->h_small);
  e->ssts.clear();
  cudaEventDestroy(e->ev0);
  cudaEventDestroy(e->ev1);
  cudaEventDestroy(e->evk0);
  cudaEventDestroy(e->evk1);
  cudaEventDestroy(e->evm0);
  cudaEventDestroy(e->evm1);
  cudaEventDestroy(e->evd0);
  cudaEventDestroy(e->evd1);
  cudaStreamDestroy(e->stream);
  delete e;
}

void* hg_engine_stream(hg_engine* e) { return e ? reinterpret_cast<void*>(e->stream) : nullptr; }
int hg_engine_set_flags(hg_engine* e, uint32_t flags) {
  HG_GUARD_BEGIN
  if (!e) return set_error(HG_ERR_INVALID, "null engine");
  std::lock_guard<std::mutex> g(e->mu);
  e->flags = flags;
  return HG_OK;
  HG_GUARD_END
}

int hg_sst_load(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* sst) {
  HG_GUARD_BEGIN
  if (!e || !schema || !sst) return set_error(HG_ERR_INVALID, "null argument");
  int rc = validate_schema(schema);
  if (rc) return rc;
  std::lock_guard<std::mutex> g(e->mu);
  CU_TRY(cudaSetDevice(e->device));
  return load_sst_locked(e, schema, sst);
  HG_GUARD_END
}

int hg_sst_unload(hg_engine* e, uint64_t id) {
  HG_GUARD_BEGIN
  if (!e) return set_error(HG_ERR_INVALID, "null engine");
  std::lock_guard<std::mutex> g(e->mu);
  auto it = e->ssts.find(id);
  if (it == e->ssts.end()) return set_error(HG_ERR_NOT_FOUND, "sst not resident");
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->stream);
  e->resident_bytes -= it->second->device_bytes;
  e->ssts.erase(it);
  return HG_OK;
  HG_GUARD_END
}

int hg_sst_resident_bytes(hg_engine* e, uint64_t* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(e->mu);
  *out = e->resident_bytes;
  return HG_OK;
  HG_GUARD_END
}

int hg_agg_export_packed(hg_engine* e, void* d_dst, uint64_t cap) {
  HG_GUARD_BEGIN
  if (!e || !d_dst) return set_error(HG_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(e->mu);
  if (cap < e->last_agg.num_groups) return set_error(HG_ERR_INVALID, "capacity smaller than the number of groups");
  CU_TRY(cudaSetDevice(e->device));
  AggOut in{const_cast<void*>(e->last_agg.d_gkey), const_cast<int64_t*>(e->last_agg.d_bucket), const_cast<uint64_t*>(e->last_agg.d_count),
            const_cast<double*>(e->last_agg.d_sum), const_cast<double*>(e->last_agg.d_min), const_cast<double*>(e->last_agg.d_max)};
  Launch L = e->L();
  k::pack_agg(L, in, e->last_gwidth, e->last_agg.num_groups, cap, static_cast<long long*>(d_dst));
  return HG_OK;
  HG_GUARD_END
}

int hg_plan_row_groups(const hg_schema_desc* schema, const uint8_t* data, uint64_t size, const hg_predicate* preds, size_t n_preds,
                       uint8_t* keep, uint32_t cap, uint32_t* num_row_groups) {
  HG_GUARD_BEGIN
  if (!data || !keep || !num_row_groups || (n_preds && !preds)) return set_error(HG_ERR_INVALID, "null argument");
  int rc = validate_schema(schema);
  if (rc) return rc;
  rc = validate_preds(schema, preds, n_preds);
  if (rc) return rc;
  hg_sst_desc d{};
  d.data = data;
  d.size = size;
  ParsedSst p;
  rc = parse_sst(schema, d, &p);
  if (rc) return rc;
  const size_t nrg = p.r->rg_rows.size();
  *num_row_groups = uint32_t(nrg);
  if (nrg > cap) return set_error(HG_ERR_INVALID, "keep[] is smaller than the number of row groups");
  uint64_t lits[MAX_PREDS];
  for (size_t i = 0; i < n_preds; i++) lits[i] = pred_literal(preds[i], schema->types[preds[i].column]);
  BloomLits bl;
  bloom_literals(schema, preds, n_preds, &bl);
  InSets sets;
  prepare_in_sets(schema, preds, n_preds, &sets);
  for (size_t g = 0; g < nrg; g++) keep[g] = rg_survives(p, g, schema, preds, lits, n_preds, sets, bl) ? 1 : 0;
  return HG_OK;
  HG_GUARD_END
}

int hg_last_stats(hg_engine* e, hg_scan_stats* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> g(e->mu);
  *out = e->stats;
  return HG_OK;
  HG_GUARD_END
}

static void end_call(hg_engine* e) {
  for (uint64_t id : e->transient_ids) e->ssts.erase(id);     // transient SSTs live in the arena: nothing to free
  e->transient_ids.clear();
}
struct CallGuard { hg_engine* e; ~CallGuard() { end_call(e); } };

// Start of every call that uses the device (the stream is idle): the previous call's statistics, staging, arena memory and with it
// the device result of its aggregate are gone
static int reset_call(hg_engine* e, uint32_t trunc_mask = 0, int trunc_gate = -1) {
  CU_TRY(cudaSetDevice(e->device));
  std::memset(&e->stats, 0, sizeof(e->stats));
  e->launches = 0;
  e->stage_cursor = 0;
  e->last_agg = hg_agg_device{};
  e->trunc_mask = trunc_mask;
  e->trunc_gate = trunc_gate;
  e->trunc_used = false;
  e->arena.reset();
  g_arena = &e->arena;
  CU_TRY(cudaEventRecord(e->ev0, e->stream));
  return HG_OK;
}

// End of a call's device work: waits for it, then its device time and launches
static int finish_call(hg_engine* e) {
  CU_TRY(cudaEventRecord(e->ev1, e->stream));
  CU_TRY(cudaStreamSynchronize(e->stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, e->ev0, e->ev1);
  e->stats.gpu_ms = ms;
  e->stats.kernel_launches = e->launches;
  return HG_OK;
}

// need_cols: the columns this call can touch (only used to select the byte ranges of non-resident SSTs)
static int begin_call(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n, const hg_predicate* preds, size_t np,
                      std::vector<uint32_t> need_cols, uint32_t trunc_mask = 0, int trunc_gate = -1) {
  int rc = validate_schema(schema);
  if (rc) return rc;
  rc = validate_preds(schema, preds, np);
  if (rc) return rc;
  if (n && !ssts) return set_error(HG_ERR_INVALID, "null sst list");
  prepare_in_sets(schema, preds, np, &e->in_sets);      // host work, ahead of the call's first event: gpu_ms stays device time
  rc = reset_call(e, trunc_mask, trunc_gate);
  if (rc) return rc;
  std::vector<size_t> pending, resident;
  for (size_t i = 0; i < n; i++) {
    if (e->ssts.count(ssts[i].id)) resident.push_back(i);
    else if (std::find_if(pending.begin(), pending.end(), [&](size_t j) { return ssts[j].id == ssts[i].id; }) == pending.end()) pending.push_back(i);
  }
  if (!pending.empty()) {
    for (uint32_t c = 0; c < schema->num_primary_keys; c++) need_cols.push_back(c);
    for (size_t i = 0; i < np; i++) need_cols.push_back(preds[i].column);
    rc = load_transient(e, schema, ssts, pending, preds, np, need_cols, n > 1, resident);
    if (rc) { end_call(e); return rc; }
  }
  return HG_OK;
}

static int scan_impl(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n, const hg_predicate* preds,
                     size_t np, const uint32_t* projection, size_t nproj, int keep_builtin, struct ArrowArrayStream* out) {
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  {
    int vrc = validate_schema(schema);     // before anything reads schema->num_columns
    if (vrc) return vrc;
  }
  std::lock_guard<std::mutex> g(e->mu);
  std::vector<uint32_t> touch;
  if (projection) for (size_t i = 0; i < nproj; i++) { if (projection[i] < schema->num_columns) touch.push_back(projection[i]); }
  else for (uint32_t c = 0; c < (keep_builtin ? schema->num_columns : schema->num_columns - 2); c++) touch.push_back(c);
  int rc = begin_call(e, schema, ssts, n, preds, np, touch);
  if (rc) return rc;
  CallGuard guard{e};
  cudaStream_t s = e->stream;
  Launch L = e->L();
  // output columns: all user columns (+ builtin when keep_builtin) or the projection (SURVEY §8 quirk 3: treated as a
  // post-merge column selection over the user columns)
  std::vector<uint32_t> out_cols;
  const uint32_t user_cols = schema->num_columns - 2;
  if (projection) {
    for (size_t i = 0; i < nproj; i++) {
      if (projection[i] >= schema->num_columns) return set_error(HG_ERR_INVALID, "projection index out of range");
      out_cols.push_back(projection[i]);
    }
  } else {
    for (uint32_t c = 0; c < (keep_builtin ? schema->num_columns : user_cols); c++) out_cols.push_back(c);
  }
  auto data = std::make_shared<StreamData>();
  for (uint32_t c : out_cols) {
    HostColumn hc;
    hc.name = col_name(schema, c);
    hc.type = schema->types[c];
    hc.width = type_width(hc.type);
    data->cols.push_back(hc);
  }
  data->batch_start.push_back(0);
  if (n == 0) { make_stream(out, data); return HG_OK; }   // EmptyRecordBatchStream (storage.rs:337-341)

  const bool append = schema->update_mode == HG_UPDATE_APPEND;
  PipelineState st;
  st.keep_order = append;
  rc = run_pipeline(e, schema, ssts, n, preds, np, out_cols, /*want_batches=*/true, &st);
  if (rc) return rc;
  const uint32_t N = st.N;
  uint32_t hc[8] = {0};
  rc = pipeline_stats(e, &st, hc);
  if (rc) return rc;
  const uint32_t R = hc[1];
  // gather + export
  DevBuf d_null;
  CU_TRY(d_null.alloc(sizeof(unsigned long long) * out_cols.size() + 16, s));
  CU_TRY(cudaMemsetAsync(d_null.p, 0, sizeof(unsigned long long) * out_cols.size() + 16, s));
  std::vector<DevBuf> gv(out_cols.size()), gb(out_cols.size()), gm(out_cols.size());
  uint64_t d2h = 0;
  // which row stands for an output row in the fixed-width columns: the run's LAST row (LastValueOperator, operator.rs:39-44) or,
  // in Append mode, its FIRST row (BytesMergeOperator takes column.slice(0, 1), operator.rs:96-100)
  DevBuf first_rows;
  const uint32_t* rep_rows = st.out_rows.as<uint32_t>();
  if (append && R > 0) {
    CU_TRY(first_rows.alloc(size_t(R) * 4 + 16, s));
    k::first_rows(L, st.order_ptr, st.out_pos.as<uint32_t>(), st.d_r, R, first_rows.as<uint32_t>());
    rep_rows = first_rows.as<uint32_t>();
  }
  for (size_t i = 0; i < out_cols.size() && R > 0; i++) {
    DecodedCol& dc = st.cols[out_cols[i]];
    HostColumn& hcx = data->cols[i];
    if (dc.type == T_BINARY) {
      // Binary: Arrow offsets by an exclusive scan of the byte lengths, then one warp per value copies the bytes.
      //   Overwrite: one value per output row (its run's last row).   Append (BytesMergeOperator, operator.rs:75-95): the values of
      //   ALL rows of a run concatenated in merged order = every surviving row's bytes laid out in merged order, offsets taken at
      //   the runs' first rows; the result is never NULL.
      const uint32_t cnt_cap = append ? N : R;                     // elements scanned (device counts: M resp. R)
      const uint32_t* src_rows = append ? st.order_ptr : st.out_rows.as<uint32_t>();
      const uint32_t* d_cnt = append ? st.d_m : st.d_r;
      DevBuf lens_scan, offs_dev, d_total;
      CU_TRY(lens_scan.alloc((size_t(cnt_cap) + 1) * 4 + 16, s));
      CU_TRY(d_total.alloc(16, s));
      k::gather_lens(L, dc.view(), src_rows, d_cnt, cnt_cap + 1, lens_scan.as<uint32_t>());
      k::exclusive_scan_u32(L, lens_scan.as<uint32_t>(), cnt_cap + 1, d_total.as<uint32_t>());
      uint32_t total = 0;
      CU_TRY(cudaMemcpyAsync(&total, d_total.p, 4, cudaMemcpyDeviceToHost, s));
      CU_TRY(cudaStreamSynchronize(s));
      if (total >= 0x7fffffffu) return set_error(HG_ERR_UNSUPPORTED, "Binary column larger than 2 GiB in one call (Arrow int32 offsets)");
      CU_TRY(gv[i].alloc(size_t(total) + 16, s));
      k::copy_var(L, dc.view(), src_rows, d_cnt, cnt_cap, lens_scan.as<uint32_t>(), gv[i].as<uint8_t>());
      const uint32_t* offs_src = lens_scan.as<uint32_t>();
      if (append) {
        CU_TRY(offs_dev.alloc((size_t(R) + 1) * 4 + 16, s));
        k::run_offsets(L, lens_scan.as<uint32_t>(), st.out_pos.as<uint32_t>(), st.d_r, st.d_m, R, offs_dev.as<uint32_t>());
        offs_src = offs_dev.as<uint32_t>();
      }
      hcx.vals = pinned_pool().alloc(size_t(total) + 16);
      hcx.offsets = static_cast<int32_t*>(pinned_pool().alloc((size_t(R) + 1) * 4 + 16));
      if (!hcx.vals || !hcx.offsets) return set_error(HG_ERR_OOM, "pinned host memory");
      if (total) CU_TRY(cudaMemcpyAsync(hcx.vals, gv[i].p, total, cudaMemcpyDeviceToHost, s));
      CU_TRY(cudaMemcpyAsync(hcx.offsets, offs_src, (size_t(R) + 1) * 4, cudaMemcpyDeviceToHost, s));
      d2h += size_t(total) + (size_t(R) + 1) * 4;
      // validity: Overwrite = the representative row's; Append = valid unless the run is ONE row whose value is NULL (a run with no
      // bytes returns its column unchanged, operator.rs:80-92; more than one such row is the reference's RecordBatch error)
      CU_TRY(gb[i].alloc(size_t(R) + 16, s));
      CU_TRY(gm[i].alloc((size_t(R) + 7) / 8 + 16, s));
      DevBuf scratch_ptrs;
      if (append) k::append_validity(L, dc.view(), st.order_ptr, st.out_pos.as<uint32_t>(), st.d_r, offs_src, R, gb[i].as<uint8_t>(), st.d_err.as<int>());
      else {
        CU_TRY(scratch_ptrs.alloc(size_t(R) * 8 + 16, s));
        k::gather_column(L, dc.view(), st.out_rows.as<uint32_t>(), st.d_r, R, scratch_ptrs.p, gb[i].as<uint8_t>());
      }
      k::pack_validity(L, gb[i].as<uint8_t>(), R, gm[i].as<uint8_t>(), d_null.as<unsigned long long>() + i);
      hcx.bitmap = static_cast<uint8_t*>(pinned_pool().alloc((size_t(R) + 7) / 8 + 16));
      if (!hcx.bitmap) return set_error(HG_ERR_OOM, "pinned host memory");
      CU_TRY(cudaMemcpyAsync(hcx.bitmap, gm[i].p, (size_t(R) + 7) / 8, cudaMemcpyDeviceToHost, s));
      d2h += (size_t(R) + 7) / 8;
      CU_TRY(cudaStreamSynchronize(s));                              // the temporaries above are popped off the arena on scope exit
      continue;
    }
    CU_TRY(gv[i].alloc(size_t(R) * dc.width + 16, s));
    bool nulls = dc.valid.p != nullptr;
    if (nulls) { CU_TRY(gb[i].alloc(size_t(R) + 16, s)); CU_TRY(gm[i].alloc((size_t(R) + 7) / 8 + 16, s)); }
    k::gather_column(L, dc.view(), rep_rows, st.d_r, R, gv[i].p, gb[i].as<uint8_t>());
    hcx.vals = pinned_pool().alloc(size_t(R) * dc.width + 16);
    if (!hcx.vals) return set_error(HG_ERR_OOM, "pinned host memory");
    CU_TRY(cudaMemcpyAsync(hcx.vals, gv[i].p, size_t(R) * dc.width, cudaMemcpyDeviceToHost, s));
    d2h += size_t(R) * dc.width;
    if (nulls) {
      k::pack_validity(L, gb[i].as<uint8_t>(), R, gm[i].as<uint8_t>(), d_null.as<unsigned long long>() + i);
      hcx.bitmap = static_cast<uint8_t*>(pinned_pool().alloc((size_t(R) + 7) / 8 + 16));
      if (!hcx.bitmap) return set_error(HG_ERR_OOM, "pinned host memory");
      CU_TRY(cudaMemcpyAsync(hcx.bitmap, gm[i].p, (size_t(R) + 7) / 8, cudaMemcpyDeviceToHost, s));
      d2h += (size_t(R) + 7) / 8;
    }
  }
  std::vector<uint32_t> bound(st.nchunks);
  if (st.nchunks && N > 0) CU_TRY(cudaMemcpyAsync(bound.data(), st.bound.p, st.nchunks * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  rc = finish_call(e);
  if (rc) return rc;
  if (append) { rc = check_device_error(e, &st); if (rc) return rc; }       // BytesMergeOperator's own failure mode (see append_validity)
  // MergeStream batch boundaries (read.rs:289-343, 349-384): batch c = outputs [bound[c-1], bound[c]); final flush = the rest
  uint32_t prev = 0;
  for (uint32_t c = 0; c < st.nchunks; c++) {
    uint32_t b = std::min(bound[c], R);
    if (b > prev) { data->batch_start.push_back(b); prev = b; }
  }
  if (R > prev) data->batch_start.push_back(R);
  e->stats.bytes_d2h = d2h + st.d2h;
  make_stream(out, data);
  return HG_OK;
}

int hg_scan_open(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                 size_t n_preds, const uint32_t* projection, size_t n_projection, int keep_builtin, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  return scan_impl(e, schema, ssts, n_ssts, preds, n_preds, projection, n_projection, keep_builtin, out);
  HG_GUARD_END
}

int hg_plan_pk_splitters(const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n, uint32_t parts, uint64_t* splitters) {
  HG_GUARD_BEGIN
  if (!ssts || !splitters || parts == 0) return set_error(HG_ERR_INVALID, "null argument");
  int rc = validate_schema(schema);
  if (rc) return rc;
  const uint32_t t0 = schema->types[0];
  struct Iv { uint64_t mn, mx, rows; };
  std::vector<Iv> ivs;
  uint64_t total = 0;
  for (size_t i = 0; i < n; i++) {
    ParsedSst p;
    rc = parse_sst(schema, ssts[i], &p);
    if (rc) return rc;
    const SstResident& r = *p.r;
    const size_t ncols = size_t(r.meta.ncols);
    for (size_t g = 0; g < r.rg_rows.size(); g++) {
      if (!r.rg_rows[g]) continue;
      const RgCol& c0 = r.rgcol[g * ncols];
      if (!c0.has_minmax) return set_error(HG_ERR_UNSUPPORTED, "pk0 statistics missing: cannot range-partition");
      ivs.push_back(Iv{c0.mn, c0.mx, r.rg_rows[g]});
      total += r.rg_rows[g];
    }
  }
  // rows of a row group are taken as evenly spread over its [min, max] of pk0 (SSTs are PK-sorted, so they nearly are);
  // splitter q = the smallest pk0 value below which at least q / parts of all rows lie under that model (bisection in the
  // order-preserving unsigned image of the column).  A balance heuristic: any splitters give a correct partition.
  const uint64_t flip = order_flip(t0);
  uint64_t lo_all = ~0ull, hi_all = 0;
  for (Iv& iv : ivs) { iv.mn ^= flip; iv.mx ^= flip; lo_all = std::min(lo_all, iv.mn); hi_all = std::max(hi_all, iv.mx); }
  auto below = [&](uint64_t x) {       // modelled number of rows with pk0 < x
    long double acc = 0;
    for (const Iv& iv : ivs) {
      if (x <= iv.mn) continue;
      if (x > iv.mx) { acc += iv.rows; continue; }
      acc += (long double)iv.rows * ((long double)(x - iv.mn) / ((long double)(iv.mx - iv.mn) + 1.0L));
    }
    return acc;
  };
  for (uint32_t q = 1; q < parts; q++) {
    uint64_t sp = hi_all;
    if (!ivs.empty()) {
      const long double want = (long double)total * q / parts;
      uint64_t a = lo_all, b = hi_all;
      while (a < b) { const uint64_t mid = a + (b - a) / 2; if (below(mid) >= want) b = mid; else a = mid + 1; }
      sp = a;
    } else sp = 0;
    splitters[q - 1] = sp ^ flip;
  }
  return HG_OK;
  HG_GUARD_END
}

// The end of hg_compact_to_sst and hg_write_batch: encodes R rows of `cols` as an SST, waits for the call's device work and writes
// the file to out_path
static int write_sst_file(hg_engine* e, const hg_schema_desc* schema, const writer::ColIn* cols, uint32_t R, const writer::WriteOpts& wo,
                          const char* out_path, uint64_t* size) {
  writer::PinnedImage img;
  int rc = writer::write_sst(e, schema, cols, R, wo, &img);
  if (!rc) rc = finish_call(e);
  if (rc) return rc;
  FILE* f = std::fopen(out_path, "wb");
  bool ok = f != nullptr;
  if (ok) ok = std::fwrite(img.p, 1, size_t(img.size), f) == size_t(img.size);
  if (f) ok = std::fclose(f) == 0 && ok;
  if (!ok) return set_error(HG_ERR_NOT_FOUND, std::string("cannot write ") + out_path);
  *size = img.size;
  return HG_OK;
}

int hg_compact_to_sst(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n, const hg_predicate* shard_preds,
                      size_t n_shard_preds, const hg_write_props* props, const char* out_path, hg_file_meta* out) {
  HG_GUARD_BEGIN
  if (!e || !props || !out_path || !out || (n_shard_preds && !shard_preds)) return set_error(HG_ERR_INVALID, "null argument");
  for (size_t i = 0; i < n_shard_preds; i++)
    if (shard_preds[i].column != 0 || shard_preds[i].op == HG_OP_IN_SET)
      return set_error(HG_ERR_INVALID, "compaction shards are ranges of the first primary-key column");
  int rc = validate_schema(schema);
  if (rc) return rc;
  writer::WriteOpts wo;                                // Binary columns and refused writer options fail here, before any device work
  rc = writer::resolve_write_opts(schema, props, &wo);
  if (rc) return rc;
  std::lock_guard<std::mutex> g(e->mu);
  std::vector<uint32_t> touch;
  for (uint32_t c = 0; c < schema->num_columns; c++) touch.push_back(c);
  rc = begin_call(e, schema, ssts, n, shard_preds, n_shard_preds, touch);
  if (rc) return rc;
  CallGuard guard{e};
  cudaStream_t s = e->stream;
  Launch L = e->L();
  std::memset(out, 0, sizeof(*out));
  for (size_t i = 0; i < n; i++) {
    if (i == 0 || ssts[i].time_start < out->time_start) out->time_start = ssts[i].time_start;
    if (i == 0 || ssts[i].time_end > out->time_end) out->time_end = ssts[i].time_end;
    out->max_sequence = std::max(out->max_sequence, ssts[i].max_sequence);
  }
  PipelineState st;
  uint32_t R = 0;
  std::vector<DevBuf> gv(schema->num_columns), gb(schema->num_columns);
  std::vector<writer::ColIn> cols(schema->num_columns);
  if (n > 0) {
    rc = run_pipeline(e, schema, ssts, n, shard_preds, n_shard_preds, touch, /*want_batches=*/false, &st);
    if (rc) return rc;
    uint32_t hc[8] = {0};
    rc = pipeline_stats(e, &st, hc);
    if (rc) return rc;
    R = hc[1];
  }
  for (uint32_t c = 0; c < schema->num_columns; c++) {
    const uint32_t width = type_width(schema->types[c]);
    cols[c] = writer::ColIn{nullptr, nullptr, schema->types[c], width};
    if (R == 0) continue;
    DecodedCol& dc = st.cols[c];
    CU_TRY(gv[c].alloc(size_t(R) * width + 16, s));
    const bool nulls = dc.valid.p != nullptr;
    if (nulls) CU_TRY(gb[c].alloc(size_t(R) + 16, s));
    k::gather_column(L, dc.view(), st.out_rows.as<uint32_t>(), st.d_r, R, gv[c].p, gb[c].as<uint8_t>());
    cols[c].vals = gv[c].p;
    cols[c].valid = nulls ? gb[c].as<uint8_t>() : nullptr;
  }
  rc = write_sst_file(e, schema, cols.data(), R, wo, out_path, &out->size);
  if (rc) return rc;
  out->num_rows = R;
  return HG_OK;
  HG_GUARD_END
}

int hg_write_batch(hg_engine* e, const hg_schema_desc* schema, const struct ArrowArray* batch, uint64_t sequence, const hg_write_props* props,
                   const char* out_path, hg_file_meta* out) {
  HG_GUARD_BEGIN
  if (!e || !batch || !props || !out_path || !out) return set_error(HG_ERR_INVALID, "null argument");
  int rc = validate_schema(schema);
  if (rc) return rc;
  const uint32_t ncols = schema->num_columns, user = ncols - 2, npk = schema->num_primary_keys;
  writer::WriteOpts wo;                                // Binary columns and refused writer options fail here, before any device work
  rc = writer::resolve_write_opts(schema, props, &wo);
  if (rc) return rc;
  if (batch->n_children != int64_t(user)) return set_error(HG_ERR_INVALID, "batch must hold the user columns of the schema");
  if (batch->length < 0 || batch->length >= 0xfffffff0ll) return set_error(HG_ERR_UNSUPPORTED, "batch larger than 2^32 rows");
  if (batch->null_count > 0) return set_error(HG_ERR_UNSUPPORTED, "NULL rows (struct-level validity) are not supported");
  const uint32_t n = uint32_t(batch->length);
  std::lock_guard<std::mutex> g(e->mu);
  rc = reset_call(e);
  if (rc) return rc;
  cudaStream_t s = e->stream;
  Launch L = e->L();
  // ---- upload the user columns (values + validity expanded to one byte per row)
  std::vector<DevBuf> vals(ncols), valid(ncols), sorted(ncols), svalid(ncols);
  std::vector<ColView> views(ncols);
  uint64_t h2d = 0;
  for (uint32_t c = 0; c < user; c++) {
    const struct ArrowArray* col = batch->children[c];
    if (!col || col->n_buffers < 2 || col->length != batch->length) return set_error(HG_ERR_INVALID, "column " + std::to_string(c) + ": not a primitive array of the batch's length");
    const uint32_t w = type_width(schema->types[c]);
    CU_TRY(vals[c].alloc(size_t(n) * w + 16, s));
    if (n) {
      if (!col->buffers[1]) return set_error(HG_ERR_INVALID, "column without a data buffer");
      CU_TRY(cudaMemcpyAsync(vals[c].p, static_cast<const uint8_t*>(col->buffers[1]) + size_t(col->offset) * w, size_t(n) * w, cudaMemcpyHostToDevice, s));
      h2d += size_t(n) * w;
    }
    const bool has_nulls = col->null_count != 0 && col->buffers[0] != nullptr;
    if (has_nulls) {
      if (c < npk) return set_error(HG_ERR_UNSUPPORTED, "NULL primary keys are not supported on the GPU path");
      const size_t nbytes = size_t((col->offset + col->length + 7) / 8);
      DevBuf bm;
      CU_TRY(bm.alloc(nbytes + 16, s));
      CU_TRY(cudaMemcpyAsync(bm.p, col->buffers[0], nbytes, cudaMemcpyHostToDevice, s));
      CU_TRY(valid[c].alloc(size_t(n) + 16, s));
      k::unpack_bitmap(L, bm.as<uint8_t>(), uint64_t(col->offset), n, valid[c].as<uint8_t>());
      bm.release();                          // arena memory: stays valid until the next call
      h2d += nbytes;
    }
    views[c] = ColView{vals[c].p, has_nulls ? valid[c].as<uint8_t>() : nullptr, schema->types[c], w, nullptr};
  }
  // ---- sort by (pk0, .., pkN-1): LSD over the key columns, last key first; every pass is a stable radix sort
  DevBuf perm, perm2, keys, keys2, counts, d_n;
  CU_TRY(perm.alloc(size_t(n) * 4 + 16, s));
  CU_TRY(perm2.alloc(size_t(n) * 4 + 16, s));
  CU_TRY(keys.alloc(size_t(n) * 8 + 16, s));
  CU_TRY(keys2.alloc(size_t(n) * 8 + 16, s));
  CU_TRY(counts.alloc(k::radix_tmp_elems(n) * 4, s));
  CU_TRY(d_n.alloc(16, s));
  k::fill_u32(L, d_n.as<uint32_t>(), n, 4);
  k::iota_u32(L, perm.as<uint32_t>(), n);
  uint32_t* pcur = perm.as<uint32_t>();
  uint32_t* palt = perm2.as<uint32_t>();
  for (int c = int(npk) - 1; c >= 0 && n > 1; c--) {
    k::column_sort_keys(L, views[c], pcur, n, keys.as<uint64_t>());
    const uint32_t t = schema->types[c];
    const int bits = (type_is_signed(t) || type_is_float(t)) ? 64 : 8 * int(type_width(t));
    if (k::radix_sort_pairs(L, keys.as<uint64_t>(), pcur, keys2.as<uint64_t>(), palt, d_n.as<uint32_t>(), n, bits, counts.as<uint32_t>())) std::swap(pcur, palt);
  }
  // ---- gather into sorted columns, append the builtin columns
  std::vector<writer::ColIn> cols(ncols);
  for (uint32_t c = 0; c < user; c++) {
    const uint32_t w = views[c].width;
    CU_TRY(sorted[c].alloc(size_t(n) * w + 16, s));
    if (views[c].valid) CU_TRY(svalid[c].alloc(size_t(n) + 16, s));
    k::gather_column(L, views[c], pcur, d_n.as<uint32_t>(), n, sorted[c].p, svalid[c].as<uint8_t>());
    cols[c] = writer::ColIn{sorted[c].p, views[c].valid ? svalid[c].as<uint8_t>() : nullptr, schema->types[c], w};
  }
  CU_TRY(sorted[user].alloc(size_t(n) * 8 + 16, s));
  k::fill_u64(L, sorted[user].as<uint64_t>(), sequence, n);
  cols[user] = writer::ColIn{sorted[user].p, nullptr, T_U64, 8};
  CU_TRY(sorted[user + 1].alloc(size_t(n) * 8 + 16, s));
  CU_TRY(svalid[user + 1].alloc(size_t(n) + 16, s));
  CU_TRY(cudaMemsetAsync(sorted[user + 1].p, 0, size_t(n) * 8 + 16, s));
  CU_TRY(cudaMemsetAsync(svalid[user + 1].p, 0, size_t(n) + 16, s));
  cols[user + 1] = writer::ColIn{sorted[user + 1].p, svalid[user + 1].as<uint8_t>(), T_U64, 8};
  uint64_t size = 0;
  rc = write_sst_file(e, schema, cols.data(), n, wo, out_path, &size);
  if (rc) return rc;
  std::memset(out, 0, sizeof(*out));
  out->size = size;
  out->num_rows = n;
  out->max_sequence = sequence;
  e->stats.bytes_h2d = h2d;
  e->stats.rows_out = n;
  return HG_OK;
  HG_GUARD_END
}

int hg_compact_open(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  // Executor::do_compaction builds the same plan with no predicate and keep_builtin = true (executor.rs:164-169)
  return scan_impl(e, schema, ssts, n_ssts, nullptr, 0, nullptr, 0, 1, out);
  HG_GUARD_END
}


// A series -> group map (hg_group_map) ready for a call: keys in the widened domain, sorted by their order key and unique, with their
// groups.  The call's predicate `pred` is `key column IN_SET keys`.
struct GroupMap {
  const uint64_t* keys = nullptr;
  const uint32_t* groups = nullptr;
  uint32_t n = 0;
  size_t pred = 0;
  std::vector<uint64_t> key_store;     // the sorted copy, when the caller's keys were not strictly increasing
  std::vector<uint32_t> group_store;
};

// An aggregate call that has passed all of its checks, with what they prepared: every stage after them reads the call from here.  Only
// the preparations (prepare_call, then take_preds, prepare_by_map or prepare_range) fill one.  The map's IN_SET predicate points into gm,
// so a call is neither copied nor moved.
struct AggCall {
  const hg_schema_desc* schema = nullptr;      // validated
  const hg_sst_desc* ssts = nullptr;
  size_t n_ssts = 0;
  const hg_agg_spec* agg = nullptr;
  std::vector<hg_predicate> preds;             // the caller's, then the map's IN_SET, then the range's time bounds
  GroupMap gm;
  const GroupMap* map = nullptr;               // &gm for a call by map
  k::RangeSpecDev rs{};                        // a range call's grid and function
  k::RangeFnSpec f{};
  int shift = 0, bits = 0;                     // a range call by map: its key (ordinal << shift) | j has `bits` bits
  AggCall() = default;
  AggCall(const AggCall&) = delete;
  AggCall& operator=(const AggCall&) = delete;
};

// The type and the name of an aggregate's group key as the call exports it: a map's u32 ordinals ("group"), else the group column's
static uint32_t group_type(const AggCall& c) {
  return c.map ? uint32_t(T_U32) : c.schema->types[c.agg->group_col];
}
static std::string group_name(const AggCall& c) {
  if (c.map) return "group";
  return c.agg->group_col >= 0 ? col_name(c.schema, uint32_t(c.agg->group_col)) : std::string();
}

// What an aggregate call requires of its spec beyond the checks every aggregate makes: a value column, a time column, one series per
// group in time order (group = pk0, time = pk1: the key is the sort prefix)
enum : uint32_t { SPEC_VALUE = 1, SPEC_TIME = 2, SPEC_SERIES = 4 };

// The spec checks of every aggregate call, all before any device work (the schema is validated).  `kind` names the call in the messages
// of what `need` requires.  A required time column that is Binary is reported as not an integer column: it is the call's time axis.
static int check_agg_spec(const hg_schema_desc* schema, const hg_agg_spec* agg, uint32_t need, const char* kind) {
  if (!agg) return set_error(HG_ERR_INVALID, "null aggregation spec");
  auto col_ok = [&](int32_t c) { return c < 0 || uint32_t(c) < schema->num_columns; };
  if (!col_ok(agg->group_col) || !col_ok(agg->ts_col) || !col_ok(agg->value_col)) return set_error(HG_ERR_INVALID, "aggregation column out of range");
  if ((need & SPEC_VALUE) && agg->value_col < 0) return set_error(HG_ERR_INVALID, std::string("a ") + kind + " aggregate needs a value column");
  if ((need & SPEC_TIME) && agg->ts_col < 0) return set_error(HG_ERR_INVALID, std::string("a ") + kind + " aggregate needs a time column");
  const bool time = (need & SPEC_TIME) || (agg->ts_col >= 0 && agg->window_ms > 0);
  for (int32_t c : {agg->group_col, (need & SPEC_TIME) ? -1 : agg->ts_col, agg->value_col})
    if (c >= 0 && schema->types[c] == T_BINARY) return set_error(HG_ERR_INVALID, "Binary columns cannot be grouped or aggregated");
  if (time && (type_is_float(schema->types[agg->ts_col]) || schema->types[agg->ts_col] == T_BINARY))
    return set_error(HG_ERR_INVALID, "time column must be an integer column");
  if (agg->mode > HG_AGG_HASH) return set_error(HG_ERR_INVALID, "aggregation mode");
  if (need & SPEC_SERIES) {
    if (schema->num_primary_keys < 2) return set_error(HG_ERR_UNSUPPORTED, std::string(kind) + " aggregate: the table needs a second primary key, the time column");
    if (agg->group_col != 0) return set_error(HG_ERR_UNSUPPORTED, std::string(kind) + " aggregate: the group column must be the first primary key (one series per group)");
    if (agg->ts_col != 1) return set_error(HG_ERR_UNSUPPORTED, std::string(kind) + " aggregate: the time column must be the second primary key (samples in time order)");
  }
  if (schema->update_mode != HG_UPDATE_OVERWRITE) return set_error(HG_ERR_UNSUPPORTED, "aggregation over an Append-mode (BytesMergeOperator) table");
  return HG_OK;
}

// The start of every aggregate call's preparation: the schema, then the call's inputs.  The spec's checks follow, and the predicates are
// taken last (take_preds, prepare_by_map, prepare_range).
static int prepare_call(AggCall* c, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_agg_spec* agg) {
  int rc = validate_schema(schema);
  if (rc) return rc;
  c->schema = schema;
  c->ssts = ssts;
  c->n_ssts = n_ssts;
  c->agg = agg;
  return HG_OK;
}

// The caller's predicates, taken into a call that adds `slots` of its own to them (the map's set: 1, the range's time bounds: 2, both: 3)
static int take_preds(AggCall* c, const hg_predicate* preds, size_t np, size_t slots) {
  static const char* const limit[] = {"more than 8 predicates", "more than 8 predicates", "more than 6 predicates (the range's time bounds take two of 8)",
                                      "more than 5 predicates (the map's set and the range's time bounds take three of 8)"};
  if (np && !preds) return set_error(HG_ERR_INVALID, "null predicates");
  if (np + slots > size_t(MAX_PREDS)) return set_error(HG_ERR_UNSUPPORTED, limit[slots]);
  c->preds.assign(preds, preds + np);
  return HG_OK;
}

// The columns an aggregate call may touch (begin_call: the byte ranges of transient SSTs); time: the call reads its time column
static std::vector<uint32_t> agg_columns(const hg_agg_spec* agg, bool time) {
  std::vector<uint32_t> cols;
  for (int32_t c : {agg->group_col, time ? agg->ts_col : -1, agg->value_col}) if (c >= 0) cols.push_back(uint32_t(c));
  return cols;
}

// The device work of one prepared call, with e->mu held: begin_call loads the transient SSTs and resets the statistics, the body runs,
// and end_call drops the transient SSTs whatever the body returns.  A call refused before begin_call leaves the last call's statistics.
// time: the call reads its time column.
static int call_frame(hg_engine* e, const AggCall& c, bool time, const std::function<int()>& body, uint32_t trunc_mask = 0, int trunc_gate = -1) {
  int rc = begin_call(e, c.schema, c.ssts, c.n_ssts, c.preds.data(), c.preds.size(), agg_columns(c.agg, time), trunc_mask, trunc_gate);
  if (rc) return rc;
  CallGuard guard{e};
  return body();
}

// Reads `bytes` of device counts that size the next stage back to the host (synchronises)
static int read_counts(hg_engine* e, void* host, const void* dev, size_t bytes) {
  CU_TRY(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, e->stream));
  CU_TRY(cudaStreamSynchronize(e->stream));
  return HG_OK;
}

// The deduplicated rows of an aggregate call cut into groups, on the general pipeline: group g is agg rows [seg[g], seg[g + 1])
// (the last one ends at *st.d_r), in stream order.  What hg_scan_aggregate (without the fused scan) and hg_scan_counter_aggregate share.
// map_groups / ordinal: map_ordinals' buffers.
struct AggGroups {
  PipelineState st;
  AggSpecDev spec;
  DevBuf head, seg, gk, gk2, vals, vals2, rcounts, map_groups, ordinal;
  const uint32_t* rows = nullptr;   // agg row t -> decoded row
  uint32_t G = 0;
};

// The map's u32 ordinal of every decoded row's group column value (group_map_kernel), as a column *key: the groups go up once; the keys
// are already on the device as the set of the map's IN_SET predicate
static int map_ordinals(hg_engine* e, const GroupMap& map, AggGroups* ag, ColView* key) {
  cudaStream_t s = e->stream;
  PipelineState& st = ag->st;
  CU_TRY(ag->map_groups.alloc(std::max<size_t>(map.n, 1) * 4, s));
  if (map.n) CU_TRY(cudaMemcpyAsync(ag->map_groups.p, map.groups, size_t(map.n) * 4, cudaMemcpyHostToDevice, s));
  e->stats.bytes_h2d += size_t(map.n) * 4;
  CU_TRY(ag->ordinal.alloc(size_t(st.N) * 4 + 16, s));
  k::group_map(e->L(), ag->spec.group, st.out_rows.as<uint32_t>(), st.d_r, st.N, e->in_sets.dev[map.pred], ag->map_groups.as<uint32_t>(), map.n,
               ag->ordinal.as<uint32_t>(), st.d_err.as<int>());
  *key = ColView{ag->ordinal.p, nullptr, T_U32, 4, nullptr};
  return HG_OK;
}

// HASH mode only differs from RUNS when the key is not a prefix of the sort order (pk0 [, bucket of pk1]) / not global: then group_rows
// radix-partitions the rows by (group value, bucket) first
static bool hash_sorted(const hg_agg_spec* agg, bool has_ts) {
  const bool prefix_key = (agg->group_col < 0 && !has_ts) || (agg->group_col == 0 && (!has_ts || agg->ts_col == 1));
  return agg->mode == HG_AGG_HASH && !prefix_key;
}

// has_ts: group by time bucket too; with_ts: decode the time column and set spec.ts even without buckets (the counter partials report
// sample times); by_map: group by the call's map's u32 ordinal of the group column instead of the column itself.  A key that is not a
// prefix of the sort order, a map's ordinal among them, is radix-partitioned by (group value, bucket) first.
static int group_rows(hg_engine* e, const AggCall& c, bool has_ts, bool with_ts, bool by_map, AggGroups* ag) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const hg_agg_spec* agg = c.agg;
  const GroupMap* map = by_map ? c.map : nullptr;
  std::vector<uint32_t> need;
  if (agg->group_col >= 0) need.push_back(uint32_t(agg->group_col));
  if (has_ts || with_ts) need.push_back(uint32_t(agg->ts_col));
  if (agg->value_col >= 0) need.push_back(uint32_t(agg->value_col));
  PipelineState& st = ag->st;
  int rc = run_pipeline(e, c.schema, c.ssts, c.n_ssts, c.preds.data(), c.preds.size(), need, /*want_batches=*/false, &st);
  if (rc) return rc;
  const uint32_t N = st.N;
  AggSpecDev& spec = ag->spec;
  std::memset(&spec, 0, sizeof(spec));
  spec.has_group = agg->group_col >= 0;
  spec.has_ts = has_ts;
  spec.has_value = agg->value_col >= 0;
  spec.window_ms = has_ts ? agg->window_ms : 1;
  if (spec.has_group) spec.group = st.cols[agg->group_col].view();
  if (has_ts || with_ts) spec.ts = st.cols[agg->ts_col].view();
  if (spec.has_value) spec.value = st.cols[agg->value_col].view();
  if (map && N > 0) {
    rc = map_ordinals(e, *map, ag, &spec.group);
    if (rc) return rc;
  }
  DevBuf &head = ag->head, &seg = ag->seg, &gk = ag->gk, &gk2 = ag->gk2, &vals = ag->vals, &vals2 = ag->vals2, &rcounts = ag->rcounts;
  const uint32_t* agg_rows = st.out_rows.as<uint32_t>();
  if ((map || hash_sorted(agg, has_ts)) && N > 0) {
    // radix partition: stable sort of the surviving rows by (group value, bucket) — bucket first, then the group value
    CU_TRY(gk.alloc(size_t(N) * 8 + 16, s));
    CU_TRY(gk2.alloc(size_t(N) * 8 + 16, s));
    CU_TRY(vals.alloc(size_t(N) * 4 + 16, s));
    CU_TRY(vals2.alloc(size_t(N) * 4 + 16, s));
    CU_TRY(rcounts.alloc(k::radix_tmp_elems(N) * sizeof(uint32_t), s));
    const uint32_t* cur = st.out_rows.as<uint32_t>();
    if (spec.has_ts) {
      k::group_sort_keys(L, spec, cur, st.d_r, N, nullptr, gk.as<uint64_t>(), vals.as<uint32_t>());
      int w = k::radix_sort_pairs(L, gk.as<uint64_t>(), vals.as<uint32_t>(), gk2.as<uint64_t>(), vals2.as<uint32_t>(), st.d_r, N, 64, rcounts.as<uint32_t>());
      if (w) std::swap(vals, vals2);
      cur = vals.as<uint32_t>();
    }
    if (spec.has_group) {
      // (vals2 receives the row ids again: the keys are recomputed in the order the first sort produced)
      k::group_sort_keys(L, spec, cur, st.d_r, N, gk.as<uint64_t>(), nullptr, vals2.as<uint32_t>());
      int w = k::radix_sort_pairs(L, gk.as<uint64_t>(), vals2.as<uint32_t>(), gk2.as<uint64_t>(), vals.as<uint32_t>(), st.d_r, N,
                                  // unsigned values occupy their native width; signed / float keys are 64-bit images
                                  (type_is_signed(spec.group.type) || type_is_float(spec.group.type)) ? 64 : 8 * int(spec.group.width),
                                  rcounts.as<uint32_t>());
      if (!w) std::swap(vals, vals2);
      cur = vals.as<uint32_t>();
    }
    agg_rows = cur;
    gk.reset();
  }
  CU_TRY(head.alloc(size_t(N) + 16, s));
  CU_TRY(seg.alloc(size_t(N) * 4 + 16, s));
  uint32_t hc[8] = {0};
  if (N > 0) {
    k::group_flags(L, spec, agg_rows, st.d_r, N, head.as<uint8_t>());
    k::clear_tail(L, head.as<uint8_t>(), st.d_r, N);
    k::compact_flags(L, head.as<uint8_t>(), N, st.tmp.as<uint32_t>(), seg.as<uint32_t>(), st.counters() + 2);
  }
  rc = pipeline_stats(e, &st, hc);
  if (rc) return rc;
  ag->rows = agg_rows;
  ag->G = hc[2];
  return HG_OK;
}

// A call by map groups by the map (always radix-partitioned, never the fused scan)
static int aggregate_core(hg_engine* e, const AggCall& c, AggBuffers* ab) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const hg_agg_spec* agg = c.agg;
  const bool has_ts = agg->ts_col >= 0 && agg->window_ms > 0;
  if (agg->group_col >= 0) { ab->gtype = group_type(c); ab->gwidth = type_width(ab->gtype); }
  if (c.n_ssts == 0) { ab->G = 0; return HG_OK; }

  // fused fast path: sorted PK-disjoint inputs, one PLAIN page per chunk, group = pk0, time = pk1
  if (!(e->flags & HG_FLAG_NO_FUSED) && !c.map && !hash_sorted(agg, has_ts)) {
    int frc = fused::try_scan_aggregate(e, c.schema, c.ssts, c.n_ssts, c.preds.data(), c.preds.size(), agg, ab);
    if (frc != fused::NOT_APPLICABLE) return frc;
  }

  AggGroups ag;
  int rc = group_rows(e, c, has_ts, /*with_ts=*/false, /*by_map=*/true, &ag);
  if (rc) return rc;
  const uint32_t G = ag.G;
  ab->G = G;
  CU_TRY(ab->alloc(G, s));
  if (G > 0) k::reduce_groups(L, ag.spec, ag.rows, ag.st.d_r, ag.seg.as<uint32_t>(), ag.st.d_g, G, ab->out());
  e->stats.groups_out = G;
  e->stats.path = 0;
  return HG_OK;
}


// Which columns may a transient load ship as compressed prefixes for this aggregate?  Only when the call has the fused scan's shape
// (fused_shape) with late materialisation and no time buckets: that kernel reads every column but pk0 only up to the row group's last
// row passing the gate column (fused_scan.cu: gate_rg_kernel, SnappyJob::partial).  *gate = the column that will be its gate.
static uint32_t aggregate_trunc_mask(const hg_engine* e, const AggCall& c, int* gate) {
  const hg_schema_desc* schema = c.schema;
  const hg_predicate* preds = c.preds.data();
  const size_t np = c.preds.size();
  const hg_agg_spec* agg = c.agg;
  *gate = -1;
  if (np == 0 || validate_preds(schema, preds, np)) return 0;   // (begin_call reports the error)
  if (e->flags & (HG_FLAG_NO_FUSED | HG_FLAG_NO_LATE_MATERIALIZATION | HG_FLAG_NO_PRUNING)) return 0;
  if (agg->ts_col >= 0 && agg->window_ms > 0) return 0;
  int extra = -1;                                    // the one predicate column besides pk0 and pk1
  for (size_t i = 0; i < np; i++) {
    const uint32_t c = preds[i].column;
    if (c >= 32) return 0;
    if (c >= 2) { if (extra >= 0 && extra != int(c)) return 0; extra = int(c); }
  }
  fused::FusedShape shape;
  if (fused::fused_shape(schema, preds, np, agg, &shape) == fused::NOT_APPLICABLE) return 0;
  *gate = shape.gate_col();
  return *gate < 0 ? 0 : ~1u;                        // everything but pk0
}

// One column of a per-group result on the device (export_groups)
struct ExportCol { std::string name; uint32_t type; const void* dev; uint32_t width; bool nullable; };

// Ends an aggregate call that returns G groups as an Arrow stream: every column crosses to pinned host memory; the nullable ones share
// the validity bitmap `bitmap` (one bit per group, on the device), which crosses once and is copied on the host.  bytes_d2h = the
// results plus pipeline_d2h.
static int export_groups(hg_engine* e, const std::vector<ExportCol>& srcs, uint32_t G, const void* bitmap, uint64_t pipeline_d2h,
                         struct ArrowArrayStream* out) {
  cudaStream_t s = e->stream;
  auto data = std::make_shared<StreamData>();
  uint64_t d2h = 0;
  const size_t bm_bytes = (size_t(G) + 7) / 8;
  uint8_t* host_bm = nullptr;                 // the validity bitmap crosses once; the other nullable columns copy it on the host
  std::vector<uint8_t*> bm_copies;
  for (auto& sc : srcs) {
    HostColumn hc;
    hc.name = sc.name;
    hc.type = sc.type;
    hc.width = sc.width;
    data->cols.push_back(hc);                 // owned by the stream from here on: an early return releases the pinned buffers
    if (!G) continue;
    HostColumn& col = data->cols.back();
    col.vals = pinned_pool().alloc(size_t(G) * sc.width + 16);
    if (!col.vals) return set_error(HG_ERR_OOM, "pinned host memory");
    CU_TRY(cudaMemcpyAsync(col.vals, sc.dev, size_t(G) * sc.width, cudaMemcpyDeviceToHost, s));
    d2h += size_t(G) * sc.width;
    if (sc.nullable) {
      col.bitmap = static_cast<uint8_t*>(pinned_pool().alloc(bm_bytes + 16));
      if (!col.bitmap) return set_error(HG_ERR_OOM, "pinned host memory");
      if (host_bm) { bm_copies.push_back(col.bitmap); continue; }
      host_bm = col.bitmap;
      CU_TRY(cudaMemcpyAsync(host_bm, bitmap, bm_bytes, cudaMemcpyDeviceToHost, s));
      d2h += bm_bytes;
    }
  }
  int rc = finish_call(e);
  if (rc) return rc;
  for (uint8_t* c : bm_copies) std::memcpy(c, host_bm, bm_bytes);
  e->stats.bytes_d2h = d2h + pipeline_d2h;
  e->stats.groups_out = G;
  data->batch_start.push_back(0);
  if (G) data->batch_start.push_back(G);
  make_stream(out, data);
  return HG_OK;
}

// The validity of n groups or windows: one byte each as the reducers write it, packed into the bitmap the stream exports.  nulls:
// pack_validity's null count, scratch, never read (the stream reports null_count -1 with a bitmap).
struct Validity {
  DevBuf valid, bitmap, nulls;
  cudaError_t alloc(uint64_t n, cudaStream_t s) {
    cudaError_t rc = valid.alloc(size_t(n) + 16, s);
    if (rc == cudaSuccess) rc = bitmap.alloc((size_t(n) + 7) / 8 + 16, s);
    if (rc == cudaSuccess) rc = nulls.alloc(16, s);
    return rc;
  }
  void pack(const Launch& L, uint32_t n) { k::pack_validity(L, valid.as<uint8_t>(), n, bitmap.as<uint8_t>(), nulls.as<unsigned long long>()); }
};

// The counter partials of n groups or windows; first_* / last_* carry the validity (NULL when it has no non-NULL value)
struct CounterCols {
  DevBuf first_ts, first_v, last_ts, last_v, inc, resets;
  cudaError_t alloc(uint64_t n, cudaStream_t s) {
    for (DevBuf* b : {&first_ts, &first_v, &last_ts, &last_v, &inc, &resets}) {
      const cudaError_t rc = b->alloc(size_t(n) * 8 + 16, s);
      if (rc != cudaSuccess) return rc;
    }
    return cudaSuccess;
  }
  void append_to(std::vector<ExportCol>* srcs) const {
    srcs->push_back({"first_ts", T_I64, first_ts.p, 8, true});
    srcs->push_back({"first_value", T_F64, first_v.p, 8, true});
    srcs->push_back({"last_ts", T_I64, last_ts.p, 8, true});
    srcs->push_back({"last_value", T_F64, last_v.p, 8, true});
    srcs->push_back({"increase", T_F64, inc.p, 8, false});
    srcs->push_back({"resets", T_U64, resets.p, 8, false});
  }
};

// quantile_0 .. quantile_(n_quantiles - 1) of n groups or windows (quantile j of group i at q[j * n + i]); each carries the validity
static void append_quantiles(std::vector<ExportCol>* srcs, const double* q, uint32_t n_quantiles, uint32_t n) {
  for (uint32_t j = 0; j < n_quantiles; j++) srcs->push_back({"quantile_" + std::to_string(j), T_F64, q + size_t(j) * n, 8, true});
}

// One aggregate call, its result as device pointers (dev: arena memory, valid until the next call) or as an Arrow stream (stream)
static int aggregate_once(hg_engine* e, const AggCall& c, uint32_t trunc_mask, int trunc_gate, hg_agg_device* dev, struct ArrowArrayStream* out) {
  return call_frame(e, c, /*time=*/true, [&]() -> int {
    AggBuffers ab;
    int rc = aggregate_core(e, c, &ab);
    if (rc) return rc;
    if (dev) {
      rc = finish_call(e);
      if (rc) return rc;
      dev->num_groups = ab.G;
      dev->d_gkey = ab.gkey.p;
      dev->d_bucket = ab.bucket.as<int64_t>();
      dev->d_count = ab.count.as<uint64_t>();
      dev->d_sum = ab.sum.as<double>();
      dev->d_min = ab.mn.as<double>();
      dev->d_max = ab.mx.as<double>();
      e->last_agg = *dev;
      e->last_gwidth = ab.gwidth;
      e->last_gtype = ab.gtype;
      for (DevBuf* b : {&ab.gkey, &ab.bucket, &ab.count, &ab.sum, &ab.mn, &ab.mx}) b->release();   // arena memory: valid until the next call
      return HG_OK;
    }
    const hg_agg_spec* agg = c.agg;
    std::vector<ExportCol> srcs;
    if (agg->group_col >= 0) srcs.push_back({group_name(c), ab.gtype, ab.gkey.p, ab.gwidth, false});
    if (agg->ts_col >= 0 && agg->window_ms > 0) srcs.push_back({"bucket", T_I64, ab.bucket.p, 8, false});
    srcs.push_back({"count", T_U64, ab.count.p, 8, false});
    if (agg->value_col >= 0) {
      srcs.push_back({"sum", T_F64, ab.sum.p, 8, false});
      srcs.push_back({"min", T_F64, ab.mn.p, 8, false});
      srcs.push_back({"max", T_F64, ab.mx.p, 8, false});
    }
    // bytes_d2h counts the result's columns only, not the general pipeline's st.d2h
    return export_groups(e, srcs, ab.G, nullptr, 0, out);
  }, trunc_mask, trunc_gate);
}

// hg_scan_aggregate and its by-map form: a call in which a compressed prefix ran out (a lopsided page, see add_prefix) is repeated with
// whole pages.  A call by map never takes the fused scan, so it ships no prefixes.
static int aggregate_call(hg_engine* e, const AggCall& c, hg_agg_device* dev, struct ArrowArrayStream* out) {
  std::lock_guard<std::mutex> g(e->mu);
  int gate = -1;
  const uint32_t mask = c.map ? 0 : aggregate_trunc_mask(e, c, &gate);
  int rc = aggregate_once(e, c, mask, gate, dev, out);
  if (rc && mask && e->trunc_used) {
    if (trace_on()) fprintf(stderr, "[transient] a compressed prefix ended before the last needed row: repeating the call with whole pages\n");
    const uint64_t wasted = e->stats.bytes_h2d;
    rc = aggregate_once(e, c, 0, -1, dev, out);
    e->stats.bytes_h2d += wasted;
    e->stats.path |= 2u;
  }
  return rc;
}

static int prepare_by_map(AggCall* c, const hg_predicate* preds, size_t np, const hg_group_map* map, size_t slots,
                          const std::function<int(const hg_group_map**)>& own = nullptr);

// The four hg_scan_aggregate[_by_map][_device] calls
static int aggregate_entry(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                           size_t n_preds, const hg_agg_spec* agg, const hg_group_map* map, bool by_map, hg_agg_device* dev,
                           struct ArrowArrayStream* out) {
  AggCall c;
  int rc = prepare_call(&c, schema, ssts, n_ssts, agg);
  if (rc) return rc;
  if (by_map) {
    rc = prepare_by_map(&c, preds, n_preds, map, 1);
  } else {
    rc = check_agg_spec(schema, agg, 0, nullptr);
    if (!rc) rc = take_preds(&c, preds, n_preds, 0);
  }
  return rc ? rc : aggregate_call(e, c, dev, out);
}

int hg_scan_aggregate_device(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                             const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg, hg_agg_device* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  return aggregate_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, nullptr, false, out, nullptr);
  HG_GUARD_END
}

int hg_scan_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                      size_t n_preds, const hg_agg_spec* agg, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  return aggregate_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, nullptr, false, nullptr, out);
  HG_GUARD_END
}

int hg_scan_counter_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                              size_t n_preds, const hg_agg_spec* agg, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  AggCall c;
  int rc = prepare_call(&c, schema, ssts, n_ssts, agg);
  if (!rc) rc = check_agg_spec(schema, agg, SPEC_VALUE | SPEC_TIME | SPEC_SERIES, "counter");
  if (!rc) rc = take_preds(&c, preds, n_preds, 0);
  if (rc) return rc;
  std::lock_guard<std::mutex> g(e->mu);
  // the general pipeline with whole pages: no fused scan, no compressed prefixes (trunc_mask 0)
  return call_frame(e, c, /*time=*/true, [&]() -> int {
    cudaStream_t s = e->stream;
    Launch L = e->L();
    const bool has_ts = agg->window_ms > 0;
    const uint32_t gtype = schema->types[agg->group_col], gwidth = type_width(gtype);
    AggGroups ag;
    if (n_ssts) {
      int rc = group_rows(e, c, has_ts, /*with_ts=*/true, /*by_map=*/false, &ag);
      if (rc) return rc;
    }
    const uint32_t G = ag.G;
    DevBuf gkey, bucket, count;
    CounterCols cc;
    Validity v;
    for (DevBuf* b : {&gkey, &bucket, &count}) CU_TRY(b->alloc(size_t(G) * 8 + 16, s));
    CU_TRY(cc.alloc(G, s));
    CU_TRY(v.alloc(G, s));
    if (G > 0) {
      CounterOut co{gkey.p, bucket.as<int64_t>(), count.as<uint64_t>(), cc.first_ts.as<int64_t>(), cc.first_v.as<double>(), cc.last_ts.as<int64_t>(),
                    cc.last_v.as<double>(), cc.inc.as<double>(), cc.resets.as<uint64_t>(), v.valid.as<uint8_t>()};
      k::reduce_counter_groups(L, ag.spec, ag.rows, ag.st.d_r, ag.seg.as<uint32_t>(), ag.st.d_g, G, co);
      v.pack(L, G);
    }
    std::vector<ExportCol> srcs{{col_name(schema, uint32_t(agg->group_col)), gtype, gkey.p, gwidth, false}};
    if (has_ts) srcs.push_back({"bucket", T_I64, bucket.p, 8, false});
    srcs.push_back({"count", T_U64, count.p, 8, false});
    cc.append_to(&srcs);
    return export_groups(e, srcs, G, v.bitmap.p, ag.st.d2h, out);
  });
  HG_GUARD_END
}

// ------------------------------------------------------------------------------------------------- quantiles
static_assert(k::kQuantileMax == HG_MAX_QUANTILES, "one bound on the quantiles of a call");

// The quantile list's checks, then the spec's, all before any device work (the schema is validated)
static int check_quantile_spec(const hg_schema_desc* schema, const hg_agg_spec* agg, const double* quantiles, uint32_t n_quantiles) {
  if (!quantiles) return set_error(HG_ERR_INVALID, "null quantiles");
  if (n_quantiles == 0 || n_quantiles > HG_MAX_QUANTILES) return set_error(HG_ERR_INVALID, "a quantile aggregate takes 1 to 16 quantiles");
  for (uint32_t i = 0; i < n_quantiles; i++)
    if (!(quantiles[i] >= 0.0 && quantiles[i] <= 1.0)) return set_error(HG_ERR_INVALID, "a quantile must lie in [0, 1]");
  return check_agg_spec(schema, agg, SPEC_VALUE, "quantile");
}

// A checked quantile list as the kernels take it
static k::QuantileSpec quantile_spec(const double* quantiles, uint32_t n_quantiles) {
  k::QuantileSpec qs;
  std::memset(&qs, 0, sizeof(qs));
  std::memcpy(qs.q, quantiles, n_quantiles * sizeof(double));
  qs.n = n_quantiles;
  return qs;
}

// The quantile tiers over n > 0 groups or windows of the value column (agg rows [0, N)): prepare(qs, qb) launches quantile_prepare over
// groups or quantile_prepare_windows over windows; then the tier sizes come back, the large tier's histogram is zeroed, the selection
// runs and the validity is packed.  Quantile j of group i lands at out[j * n + i].  large_cap: the capacity of the large tier.
static int quantile_stage(hg_engine* e, const double* quantiles, uint32_t n_quantiles, uint32_t value_type, uint32_t N, uint32_t n,
                          size_t large_cap, double* out, Validity* v,
                          const std::function<void(const k::QuantileSpec&, const k::QuantileBufs&)>& prepare) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const k::QuantileSpec qs = quantile_spec(quantiles, n_quantiles);
  DevBuf flags, ctmp, idx, keys, list, large, hist, counters;
  CU_TRY(flags.alloc(size_t(N) + 16, s));
  CU_TRY(ctmp.alloc(k::compact_tmp_elems(N) * 4 + 16, s));
  CU_TRY(idx.alloc(size_t(N) * 4 + 16, s));
  CU_TRY(keys.alloc(size_t(N) * 8 + 16, s));
  CU_TRY(list.alloc(size_t(n) * sizeof(k::QuantileGroup) + 16, s));
  CU_TRY(large.alloc(large_cap * sizeof(k::QuantileLarge), s));
  CU_TRY(counters.alloc(k::kQuantileCounters * 4, s));
  CU_TRY(cudaMemsetAsync(counters.p, 0, k::kQuantileCounters * 4, s));
  k::QuantileBufs qb{flags.as<uint8_t>(), ctmp.as<uint32_t>(), idx.as<uint32_t>(), keys.as<uint64_t>(), list.as<k::QuantileGroup>(),
                     large.as<k::QuantileLarge>(), nullptr, counters.as<uint32_t>(), out, v->valid.as<uint8_t>()};
  prepare(qs, qb);
  // the tier sizes (a few words) decide which selection kernels run
  uint32_t hc[k::kQuantileCounters];
  int rc = read_counts(e, hc, counters.p, sizeof(hc));
  if (rc) return rc;
  CU_TRY(hist.alloc(k::quantile_hist_elems(hc[k::QC_LARGE]) * 4 + 16, s));
  CU_TRY(cudaMemsetAsync(hist.p, 0, k::quantile_hist_elems(hc[k::QC_LARGE]) * 4, s));
  qb.hist = hist.as<uint32_t>();
  k::quantile_select(L, qs, value_type, n, hc, qb);
  v->pack(L, n);
  return HG_OK;
}

// hg_scan_quantile_aggregate and its by-map form: the general pipeline with whole pages (no fused scan, no compressed prefixes:
// trunc_mask 0) and the quantile kernels
static int quantile_entry(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                          size_t n_preds, const hg_agg_spec* agg, const hg_group_map* map, bool by_map, const double* quantiles,
                          uint32_t n_quantiles, struct ArrowArrayStream* out) {
  AggCall c;
  int rc = prepare_call(&c, schema, ssts, n_ssts, agg);
  if (!rc) rc = check_quantile_spec(schema, agg, quantiles, n_quantiles);
  if (!rc) rc = by_map ? prepare_by_map(&c, preds, n_preds, map, 1) : take_preds(&c, preds, n_preds, 0);
  if (rc) return rc;
  const bool has_ts = agg->ts_col >= 0 && agg->window_ms > 0;
  std::lock_guard<std::mutex> g(e->mu);
  return call_frame(e, c, has_ts, [&]() -> int {
    cudaStream_t s = e->stream;
    Launch L = e->L();
    AggGroups ag;
    if (n_ssts) {
      int rc = group_rows(e, c, has_ts, /*with_ts=*/false, /*by_map=*/true, &ag);
      if (rc) return rc;
    }

    const uint32_t G = ag.G, N = ag.st.N;
    // key, bucket and count as hg_scan_aggregate computes them (reduce_groups without a value: sum / min / max are not read)
    AggBuffers ab;
    CU_TRY(ab.alloc(G, s));
    DevBuf qout;
    Validity v;
    CU_TRY(qout.alloc(size_t(G) * n_quantiles * 8 + 16, s));
    CU_TRY(v.alloc(G, s));
    if (G > 0) {
      AggSpecDev kspec = ag.spec;
      kspec.has_value = 0;
      k::reduce_groups(L, kspec, ag.rows, ag.st.d_r, ag.seg.as<uint32_t>(), ag.st.d_g, G, ab.out());
      int rc = quantile_stage(e, quantiles, n_quantiles, schema->types[agg->value_col], N, G, k::quantile_large_cap(N), qout.as<double>(), &v,
                              [&](const k::QuantileSpec& qs, const k::QuantileBufs& qb) {
                                k::quantile_prepare(L, ag.spec.value, ag.rows, ag.st.d_r, N, ag.seg.as<uint32_t>(), ag.st.d_g, G, qs, qb);
                              });
      if (rc) return rc;
    }
    std::vector<ExportCol> srcs;
    if (agg->group_col >= 0) srcs.push_back({group_name(c), group_type(c), ab.gkey.p, type_width(group_type(c)), false});
    if (has_ts) srcs.push_back({"bucket", T_I64, ab.bucket.p, 8, false});
    srcs.push_back({"count", T_U64, ab.count.p, 8, false});
    append_quantiles(&srcs, qout.as<double>(), n_quantiles, G);
    return export_groups(e, srcs, G, v.bitmap.p, ag.st.d2h, out);
  });
}

int hg_scan_quantile_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                               size_t n_preds, const hg_agg_spec* agg, const double* quantiles, uint32_t n_quantiles,
                               struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  return quantile_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, nullptr, false, quantiles, n_quantiles, out);
  HG_GUARD_END
}

// ------------------------------------------------------------------------------------------------- aggregates by label group
// The by-map preparation, all before any device work and before any read of the map's arrays: the map's pointers, the spec (a quantile
// call has checked its own already), the key column and the predicates, with `slots` taken by the call's own (the map's set: 1, with a
// range's time bounds: 3).  Then the entry's own checks (own), which may give the map to prepare in place of the caller's (the histogram
// call's dense map).  Then the map sorted by its keys' order keys with its duplicates removed (a key mapped to two groups is refused),
// and the call's predicates: the caller's, then `group_col IN_SET keys`.  An index lookup usually delivers its series in order: one pass
// checks for "strictly increasing" and such a map is used in place; prepare_in_sets then finds the set increasing too and does not sort
// it again.
static int prepare_by_map(AggCall* c, const hg_predicate* preds, size_t np, const hg_group_map* map, size_t slots,
                          const std::function<int(const hg_group_map**)>& own) {
  const hg_schema_desc* schema = c->schema;
  const hg_agg_spec* agg = c->agg;
  if (!map) return set_error(HG_ERR_INVALID, "null group map");
  if (map->count > HG_MAX_IN_SET) return set_error(HG_ERR_INVALID, "group map: more than HG_MAX_IN_SET keys");
  if (map->count && (!map->keys || !map->groups)) return set_error(HG_ERR_INVALID, "group map: null keys or groups");
  int rc = check_agg_spec(schema, agg, 0, nullptr);
  if (rc) return rc;
  if (agg->group_col < 0) return set_error(HG_ERR_INVALID, "an aggregate by map needs its key column as group_col");
  if (type_is_float(schema->types[agg->group_col]))
    return set_error(HG_ERR_UNSUPPORTED, "group map on a float column: set predicates are implemented for integer columns only");
  rc = take_preds(c, preds, np, slots);
  if (rc) return rc;
  if (own) {
    rc = own(&map);
    if (rc) return rc;
  }

  const auto t0 = HostClock::now();
  GroupMap* gm = &c->gm;
  const uint64_t flip = order_flip(schema->types[agg->group_col]);
  const uint32_t n = map->count;
  bool increasing = true;
  for (uint32_t j = 1; j < n && increasing; j++) increasing = (map->keys[j] ^ flip) > (map->keys[j - 1] ^ flip);
  if (increasing) {
    gm->keys = map->keys;
    gm->groups = map->groups;
    gm->n = n;
  } else {
    std::vector<std::pair<uint64_t, uint32_t>> kv(n);
    for (uint32_t j = 0; j < n; j++) kv[j] = {map->keys[j] ^ flip, map->groups[j]};
    std::sort(kv.begin(), kv.end());
    gm->key_store.reserve(n);
    gm->group_store.reserve(n);
    for (uint32_t j = 0; j < n; j++) {
      if (j && kv[j].first == kv[j - 1].first) {
        if (kv[j].second != kv[j - 1].second) return set_error(HG_ERR_INVALID, "group map: a key mapped to two different groups");
        continue;
      }
      gm->key_store.push_back(kv[j].first ^ flip);
      gm->group_store.push_back(kv[j].second);
    }
    gm->keys = gm->key_store.data();
    gm->groups = gm->group_store.data();
    gm->n = uint32_t(gm->key_store.size());
  }
  if (trace_on())
    fprintf(stderr, "[group_map] %u keys -> %u, %s, %.0f us\n", n, gm->n, increasing ? "already sorted" : "sorted on the host",
            elapsed_us(t0, HostClock::now()));
  hg_predicate p;
  std::memset(&p, 0, sizeof(p));
  p.column = uint32_t(agg->group_col);
  p.op = HG_OP_IN_SET;
  p.in_values = gm->keys;
  p.in_count = gm->n;
  c->preds.push_back(p);
  gm->pred = np;
  c->map = gm;
  return HG_OK;
}

int hg_scan_aggregate_by_map(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                             size_t n_preds, const hg_agg_spec* agg, const hg_group_map* map, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  return aggregate_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, map, true, nullptr, out);
  HG_GUARD_END
}

int hg_scan_aggregate_by_map_device(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                                    const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg, const hg_group_map* map,
                                    hg_agg_device* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  return aggregate_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, map, true, out, nullptr);
  HG_GUARD_END
}

int hg_scan_quantile_aggregate_by_map(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts,
                                      const hg_predicate* preds, size_t n_preds, const hg_agg_spec* agg, const hg_group_map* map,
                                      const double* quantiles, uint32_t n_quantiles, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  return quantile_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, map, true, quantiles, n_quantiles, out);
  HG_GUARD_END
}

// ------------------------------------------------------------------------------------------------- range windows
// A range call's checks, all before any device work (the schema is validated): the counter call's key shape and value, then the grid.
// *rs = the grid as the kernels take it.
static int check_range_spec(const hg_schema_desc* schema, const hg_agg_spec* agg, const hg_range_spec* range, k::RangeSpecDev* rs) {
  if (!range) return set_error(HG_ERR_INVALID, "null range spec");
  int rc = check_agg_spec(schema, agg, SPEC_VALUE | SPEC_TIME | SPEC_SERIES, "counter");
  if (rc) return rc;
  if (agg->window_ms > 0) return set_error(HG_ERR_INVALID, "a range aggregate takes its windows from the range spec: window_ms must be <= 0");
  if (schema->types[agg->ts_col] == T_U64)
    return set_error(HG_ERR_UNSUPPORTED, "range aggregate on a u64 time column: times from 2^63 on do not keep their order in i64");
  const hg_range_spec& r = *range;
  if (r.range_ms <= 0) return set_error(HG_ERR_INVALID, "range spec: range_ms must be > 0");
  if (r.start_ms > r.end_ms) return set_error(HG_ERR_INVALID, "range spec: start_ms > end_ms");
  if (r.start_ms != r.end_ms && r.step_ms <= 0) return set_error(HG_ERR_INVALID, "range spec: step_ms must be > 0");
  // with both in i64, every intermediate of the window arithmetic (ts - start, ts + range - 1 - start, start + j * step) is in i64 too
  const __int128 lo = __int128(r.start_ms) - r.range_ms, span = (__int128(r.end_ms) - r.start_ms) + r.range_ms;
  if (lo < __int128(INT64_MIN) || span > __int128(INT64_MAX))
    return set_error(HG_ERR_INVALID, "range spec: start_ms - range_ms or (end_ms - start_ms) + range_ms does not fit in i64");
  const int64_t step = r.start_ms == r.end_ms ? 1 : r.step_ms;
  const uint64_t n = uint64_t(r.end_ms - r.start_ms) / uint64_t(step) + 1;
  if (n > HG_MAX_RANGE_STEPS) return set_error(HG_ERR_INVALID, "range spec: more than HG_MAX_RANGE_STEPS steps");
  *rs = k::RangeSpecDev{r.start_ms, step, r.range_ms, uint32_t(n), 0};
  return HG_OK;
}

// The call's time bounds after its other predicates:  ts > start - range  and  ts <= end.  A bound that excludes nothing in the time
// column's domain is left out; an upper bound below an unsigned column's domain becomes `ts < 0`, which no row passes.
static void range_preds(AggCall* c, const hg_range_spec& r) {
  const uint32_t t = c->schema->types[c->agg->ts_col];
  const bool sgn = type_is_signed(t);
  const int bits = 8 * int(type_width(t));          // a u64 time column is refused: an unsigned domain here has at most 32 bits
  const int64_t tmin = !sgn ? 0 : bits == 64 ? INT64_MIN : -(int64_t(1) << (bits - 1));
  const int64_t tmax = bits == 64 ? INT64_MAX : sgn ? (int64_t(1) << (bits - 1)) - 1 : (int64_t(1) << bits) - 1;
  auto bound = [&](uint32_t op, int64_t lit) {
    hg_predicate p;
    std::memset(&p, 0, sizeof(p));
    p.column = uint32_t(c->agg->ts_col);
    p.op = op;
    if (sgn) p.i64 = lit;
    else p.u64 = uint64_t(lit);
    c->preds.push_back(p);
  };
  const int64_t after = r.start_ms - r.range_ms;    // rows need ts > after
  if (after >= tmin) bound(HG_OP_GT, after);
  if (r.end_ms < tmax) {
    if (!sgn && r.end_ms < 0) bound(HG_OP_LT, 0);
    else bound(HG_OP_LE, r.end_ms);
  }
}

static int bit_length(uint64_t x) { return x ? 64 - __builtin_clzll(x) : 0; }

static constexpr uint32_t kNoFn = ~0u;   // a range call without a function (hg_scan_range_[quantile_]aggregate)

// The range preparation, all before any device work: the function, the spec and the grid, the predicates with the two slots of the time
// bounds, then with a map the by-map preparation (own: see prepare_by_map), then the time bounds after the other predicates, the
// function as the kernels take it and the by-map key (ordinal << shift) | j: the fewest bits that hold every ordinal of the map and every
// step (j < n <= 2^24).
static int prepare_range(AggCall* c, const hg_predicate* preds, size_t np, const hg_range_spec* range, uint32_t fn, const hg_group_map* map,
                         const std::function<int(const hg_group_map**)>& own = nullptr) {
  if (fn != kNoFn && fn >= k::kFnCount) return set_error(HG_ERR_INVALID, "range function: fn is not an hg_range_fn");
  int rc = check_range_spec(c->schema, c->agg, range, &c->rs);
  if (!rc) rc = take_preds(c, preds, np, 2);
  if (!rc && map) rc = prepare_by_map(c, preds, np, map, 3, own);
  if (rc) return rc;
  range_preds(c, *range);
  const int64_t R = range->range_ms;
  c->f = k::RangeFnSpec{R, double(R / 1000) + double((R % 1000) * 1000000) / 1e9, fn, 0};
  c->shift = bit_length(c->rs.n - 1);
  if (c->map) {
    uint32_t max_ordinal = 0;
    for (uint32_t i = 0; i < c->map->n; i++) max_ordinal = std::max(max_ordinal, c->map->groups[i]);
    c->bits = c->shift + bit_length(max_ordinal);
  }
  return HG_OK;
}

// The windows of a range call on the general pipeline with whole pages (no fused scan, no compressed prefixes): one group per series, the
// gathered arrays (rb), the window count W and every window's rows, time and key (gkey).  The key is the series column, or with a map
// the series' u32 ordinal: map_ordinals writes one per row, and range_windows reads them through a ColView as it reads a column.
struct RangeState {
  AggGroups ag;
  uint64_t W = 0, members = 0;
  DevBuf ts, v, ok, off, wsum, msum, totals, win_lo, win_hi, win_t, gkey;
  k::RangeBufs rb{};
  uint32_t gwidth = 0;
};

static int range_stage(hg_engine* e, const AggCall& c, RangeState* r) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const k::RangeSpecDev& rs = c.rs;
  AggGroups& ag = r->ag;
  if (c.n_ssts) {
    // one group per series: the counter call's RUNS grouping over pk0, with the time column decoded (a map's ordinals do not group: two
    // series of one label group stay two series)
    int rc = group_rows(e, c, /*has_ts=*/false, /*with_ts=*/true, /*by_map=*/false, &ag);
    if (rc) return rc;
  }
  const uint32_t G = ag.G, N = ag.st.N;
  uint64_t& W = r->W;
  DevBuf &ts = r->ts, &v = r->v, &ok = r->ok, &off = r->off, &wsum = r->wsum, &msum = r->msum, &totals = r->totals;
  k::RangeBufs& rb = r->rb;
  ColView key = ag.spec.group;
  if (c.map && G > 0) {
    const int rc = map_ordinals(e, *c.map, &ag, &key);
    if (rc) return rc;
  }
  if (G > 0) {
    CU_TRY(ts.alloc(size_t(N) * 8 + 16, s));
    CU_TRY(v.alloc(size_t(N) * 8 + 16, s));
    CU_TRY(ok.alloc(size_t(N) + 16, s));
    CU_TRY(off.alloc(size_t(N) * 4 + 16, s));
    CU_TRY(wsum.alloc(k::range_block_elems(N) * 8, s));
    CU_TRY(msum.alloc(k::range_block_elems(N) * 8, s));
    CU_TRY(totals.alloc(16, s));
    rb = k::RangeBufs{ts.as<int64_t>(), v.as<double>(), ok.as<uint8_t>(), off.as<uint32_t>(), wsum.as<uint64_t>(), msum.as<uint64_t>(),
                      totals.as<uint64_t>()};
    k::range_count(L, rs, ag.spec.ts, ag.spec.value, ag.rows, ag.st.d_r, N, ag.head.as<uint8_t>(), rb);
    // the window count sizes the rest (16 bytes: the windows and the sum of their lengths)
    uint64_t ht[2];
    int rc = read_counts(e, ht, totals.p, sizeof(ht));
    if (rc) return rc;
    W = ht[0];
    r->members = ht[1];
    if (c.map) {
      rc = check_device_error(e, &ag.st);     // a row of the map's set without a group
      if (rc) return rc;
    }
    if (W > UINT32_MAX) return set_error(HG_ERR_OOM, "range aggregate: more than 2^32 - 1 windows in the result");
  }
  r->gwidth = c.map ? 4 : type_width(c.schema->types[c.agg->group_col]);
  CU_TRY(r->win_lo.alloc(size_t(W) * 4 + 16, s));
  CU_TRY(r->win_hi.alloc(size_t(W) * 4 + 16, s));
  CU_TRY(r->win_t.alloc(size_t(W) * 8 + 16, s));
  CU_TRY(r->gkey.alloc(size_t(W) * r->gwidth + 16, s));
  k::range_windows(L, rs, ag.st.d_r, N, ag.head.as<uint8_t>(), ag.seg.as<uint32_t>(), G, key, ag.rows, uint32_t(W), rb,
                   k::RangeWindows{r->win_lo.as<uint32_t>(), r->win_hi.as<uint32_t>(), r->win_t.as<int64_t>(), r->gkey.p});
  return HG_OK;
}

// The range windows, then the reducers (quantiles == nullptr) or the quantile tiers
static int range_call(hg_engine* e, const AggCall& c, const double* quantiles, uint32_t n_quantiles, struct ArrowArrayStream* out) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const hg_schema_desc* schema = c.schema;
  const hg_agg_spec* agg = c.agg;
  RangeState r;
  int rc = range_stage(e, c, &r);
  if (rc) return rc;
  AggGroups& ag = r.ag;
  const uint32_t N = ag.st.N, W = uint32_t(r.W);      // range_stage refuses more than 2^32 - 1 windows
  const uint32_t* win_lo = r.win_lo.as<uint32_t>();
  const uint32_t* win_hi = r.win_hi.as<uint32_t>();

  std::vector<ExportCol> srcs{{col_name(schema, uint32_t(agg->group_col)), schema->types[agg->group_col], r.gkey.p, r.gwidth, false},
                              {"t", T_I64, r.win_t.p, 8, false}};
  DevBuf count;
  Validity v;
  CU_TRY(count.alloc(size_t(W) * 8 + 16, s));
  CU_TRY(v.alloc(W, s));
  srcs.push_back({"count", T_U64, count.p, 8, false});
  if (!quantiles) {
    DevBuf sum, mn, mx;
    CounterCols cc;
    for (DevBuf* b : {&sum, &mn, &mx}) CU_TRY(b->alloc(size_t(W) * 8 + 16, s));
    CU_TRY(cc.alloc(W, s));
    if (W > 0) {
      k::RangeOut ro{count.as<uint64_t>(), sum.as<double>(), mn.as<double>(), mx.as<double>(), cc.first_ts.as<int64_t>(), cc.first_v.as<double>(),
                     cc.last_ts.as<int64_t>(), cc.last_v.as<double>(), cc.inc.as<double>(), cc.resets.as<uint64_t>(), v.valid.as<uint8_t>()};
      k::reduce_range_windows(L, r.rb, win_lo, win_hi, W, ro);
      v.pack(L, W);
    }
    srcs.push_back({"sum", T_F64, sum.p, 8, false});
    srcs.push_back({"min", T_F64, mn.p, 8, false});
    srcs.push_back({"max", T_F64, mx.p, 8, false});
    cc.append_to(&srcs);
    return export_groups(e, srcs, W, v.bitmap.p, ag.st.d2h, out);
  }

  DevBuf qout;
  CU_TRY(qout.alloc(size_t(W) * n_quantiles * 8 + 16, s));
  if (W > 0) {
    // Windows overlap, so quantile_large_cap (disjoint groups) does not bound the large tier: at most members / (kQuantileMediumMax + 1)
    // windows are large, and their chunks (the low word of QC_LARGE_CHUNKS) number at most members / kQuantileChunk + W
    if (r.members / k::kQuantileChunk + r.W > UINT32_MAX)
      return set_error(HG_ERR_OOM, "range quantile aggregate: the windows' key chunks exceed 2^32 - 1");
    const size_t n_large = size_t(std::min<uint64_t>(r.W, r.members / (k::kQuantileMediumMax + 1))) + 1;
    rc = quantile_stage(e, quantiles, n_quantiles, schema->types[agg->value_col], N, W, n_large, qout.as<double>(), &v,
                        [&](const k::QuantileSpec& qs, const k::QuantileBufs& qb) {
                          k::quantile_prepare_windows(L, ag.spec.value, ag.rows, ag.st.d_r, N, win_lo, win_hi, W, qs, qb, count.as<uint64_t>());
                        });
    if (rc) return rc;
  }
  append_quantiles(&srcs, qout.as<double>(), n_quantiles, W);
  return export_groups(e, srcs, W, v.bitmap.p, ag.st.d2h, out);
}

static int range_entry(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds, size_t n_preds,
                       const hg_agg_spec* agg, const hg_range_spec* range, const double* quantiles, uint32_t n_quantiles, struct ArrowArrayStream* out) {
  AggCall c;
  int rc = prepare_call(&c, schema, ssts, n_ssts, agg);
  if (!rc && (quantiles || n_quantiles)) rc = check_quantile_spec(schema, agg, quantiles, n_quantiles);
  if (!rc) rc = prepare_range(&c, preds, n_preds, range, kNoFn, nullptr);
  if (rc) return rc;
  std::lock_guard<std::mutex> g(e->mu);
  return call_frame(e, c, /*time=*/true, [&]() -> int { return range_call(e, c, quantiles, n_quantiles, out); });
}

int hg_scan_range_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                            size_t n_preds, const hg_agg_spec* agg, const hg_range_spec* range, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  return range_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, range, nullptr, 0, out);
  HG_GUARD_END
}

int hg_scan_range_quantile_aggregate(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                                     size_t n_preds, const hg_agg_spec* agg, const hg_range_spec* range, const double* quantiles,
                                     uint32_t n_quantiles, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  if (!quantiles) return set_error(HG_ERR_INVALID, "null quantiles");
  return range_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, range, quantiles, n_quantiles, out);
  HG_GUARD_END
}

// ------------------------------------------------------------------------------------------------- range functions
static_assert(k::kFnRate == uint32_t(HG_FN_RATE) && k::kFnIdelta == uint32_t(HG_FN_IDELTA) && k::kFnChanges == uint32_t(HG_FN_CHANGES) &&
              k::kFnLastOverTime == uint32_t(HG_FN_LAST_OVER_TIME) && k::kFnCount == uint32_t(HG_FN_LAST_OVER_TIME) + 1,
              "one numbering of the range functions");

// The range windows of a range function call (range_stage, with the map's ordinal as the windows' key), the function of every window
// and the windows with a value: idx[0 .. cnt[0]).  cnt: four device counts, the others for the stages after this one.
struct RangeFnValues {
  RangeState r;
  DevBuf value, valid, idx, ctmp, cnt;
  uint32_t W = 0;
  uint32_t* d_n() { return cnt.as<uint32_t>(); }
};

static int range_fn_values(hg_engine* e, const AggCall& c, RangeFnValues* fv) {
  cudaStream_t s = e->stream;
  RangeState& r = fv->r;
  int rc = range_stage(e, c, &r);
  if (rc) return rc;
  const uint32_t W = fv->W = uint32_t(r.W);              // range_stage refuses more than 2^32 - 1 windows
  CU_TRY(fv->value.alloc(size_t(W) * 8 + 16, s));
  CU_TRY(fv->valid.alloc(size_t(W) + 16, s));
  CU_TRY(fv->idx.alloc(size_t(W) * 4 + 16, s));
  CU_TRY(fv->ctmp.alloc(k::compact_tmp_elems(W) * 4 + 16, s));
  CU_TRY(fv->cnt.alloc(16, s));
  CU_TRY(cudaMemsetAsync(fv->cnt.p, 0, 16, s));
  if (W > 0) {
    Launch L = e->L();
    k::range_function(L, c.f, r.rb, r.win_lo.as<uint32_t>(), r.win_hi.as<uint32_t>(), r.win_t.as<int64_t>(), W, fv->value.as<double>(),
                      fv->valid.as<uint8_t>());
    k::compact_flags(L, fv->valid.as<uint8_t>(), W, fv->ctmp.as<uint32_t>(), fv->idx.as<uint32_t>(), fv->d_n());
  }
  return HG_OK;
}

// The device work of every range function call, with its own tail after the windows with a value
static int range_fn_call(hg_engine* e, const AggCall& c, const std::function<int(RangeFnValues&)>& tail) {
  std::lock_guard<std::mutex> g(e->mu);
  return call_frame(e, c, /*time=*/true, [&]() -> int {
    RangeFnValues fv;
    const int rc = range_fn_values(e, c, &fv);
    return rc ? rc : tail(fv);
  });
}

// The windows with a value cut into runs per (key, t): sort_keys(keys, vals) writes a sort key of `bits` bits and the window for each of
// them, or without sort_keys the call's by-map key (ordinal << c.shift) | j of c.bits bits.  One stable radix_sort_pairs orders them (the
// windows of one key keep the order of fv->idx, their series order unless the caller has reordered it), group_flags cuts them where the
// key changes: run r starts at seg[r], the sorted windows are vals.  cnt[1] = the runs.
struct RangeFnSegments {
  DevBuf keys, keys2, vals, vals2, rcounts, head, seg;
};

static int range_fn_segments(hg_engine* e, const AggCall& c, RangeFnValues* fv, RangeFnSegments* sums, int bits = 0,
                             const std::function<void(uint64_t*, uint32_t*)>& sort_keys = nullptr) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const uint32_t W = fv->W;
  uint32_t* d_n = fv->d_n();
  if (W == 0) return HG_OK;
  DevBuf &keys = sums->keys, &keys2 = sums->keys2, &vals = sums->vals, &vals2 = sums->vals2;
  CU_TRY(keys.alloc(size_t(W) * 8 + 16, s));
  CU_TRY(keys2.alloc(size_t(W) * 8 + 16, s));
  CU_TRY(vals.alloc(size_t(W) * 4 + 16, s));
  CU_TRY(vals2.alloc(size_t(W) * 4 + 16, s));
  CU_TRY(sums->rcounts.alloc(k::radix_tmp_elems(W) * sizeof(uint32_t), s));
  CU_TRY(sums->head.alloc(size_t(W) + 16, s));
  CU_TRY(sums->seg.alloc(size_t(W) * 4 + 16, s));
  if (sort_keys) {
    sort_keys(keys.as<uint64_t>(), vals.as<uint32_t>());
  } else {
    k::range_fn_sort_keys(L, fv->idx.as<uint32_t>(), d_n, W, fv->r.gkey.as<uint32_t>(), fv->r.win_t.as<int64_t>(), c.rs.start, c.rs.step, c.shift,
                          keys.as<uint64_t>(), vals.as<uint32_t>());
    bits = c.bits;
  }
  // stable: the windows of one (key, t) keep their series order
  if (k::radix_sort_pairs(L, keys.as<uint64_t>(), vals.as<uint32_t>(), keys2.as<uint64_t>(), vals2.as<uint32_t>(), d_n, W, bits,
                          sums->rcounts.as<uint32_t>())) {
    std::swap(keys, keys2);
    std::swap(vals, vals2);
  }
  AggSpecDev cut;
  std::memset(&cut, 0, sizeof(cut));
  cut.has_group = 1;
  cut.group = ColView{keys.p, nullptr, T_U64, 8, nullptr};
  cut.window_ms = 1;
  k::group_flags(L, cut, nullptr, d_n, W, sums->head.as<uint8_t>());
  k::clear_tail(L, sums->head.as<uint8_t>(), d_n, W);
  k::compact_flags(L, sums->head.as<uint8_t>(), W, fv->ctmp.as<uint32_t>(), sums->seg.as<uint32_t>(), d_n + 1);
  return HG_OK;
}

// range_fn_segments, then reduce_groups_kernel reduces each run over the window arrays: group = the window's u32 ordinal, bucket = t,
// count / sum / min / max of the function's values, the sum in series order.
struct RangeFnSums : RangeFnSegments {
  AggBuffers ab;
};

static int range_fn_sums(hg_engine* e, const AggCall& c, RangeFnValues* fv, RangeFnSums* sums, int bits = 0,
                         const std::function<void(uint64_t*, uint32_t*)>& sort_keys = nullptr) {
  const uint32_t W = fv->W;
  uint32_t* d_n = fv->d_n();
  CU_TRY(sums->ab.alloc(W, e->stream));
  if (W == 0) return HG_OK;
  int rc = range_fn_segments(e, c, fv, sums, bits, sort_keys);
  if (rc) return rc;
  Launch L = e->L();
  // hg_scan_aggregate's reducer over the window arrays: group = the ordinal, bucket = t (window_ms 1), value = the function's value
  AggSpecDev red;
  std::memset(&red, 0, sizeof(red));
  red.has_group = red.has_ts = red.has_value = 1;
  red.window_ms = 1;
  red.group = ColView{fv->r.gkey.p, nullptr, T_U32, 4, nullptr};
  red.ts = ColView{fv->r.win_t.p, nullptr, T_I64, 8, nullptr};
  red.value = ColView{fv->value.p, nullptr, T_F64, 8, nullptr};
  k::reduce_groups(L, red, sums->vals.as<uint32_t>(), d_n, sums->seg.as<uint32_t>(), d_n + 1, W, sums->ab.out());
  return HG_OK;
}

// The windows with a value, then per series (no map) those windows gathered, or per (group, t) their count / sum / min / max
// (range_fn_sums with the by-map key), so that a group's sum takes its series in stream order.
static int range_function_tail(hg_engine* e, const AggCall& c, RangeFnValues& fv, struct ArrowArrayStream* out) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const RangeState& r = fv.r;
  uint32_t* d_n = fv.d_n();
  uint32_t hn[2] = {0, 0};
  if (!c.map) {
    int rc = read_counts(e, hn, d_n, sizeof(hn));
    if (rc) return rc;
    const uint32_t n = hn[0], gtype = c.schema->types[c.agg->group_col];
    DevBuf key_out, t_out, v_out;
    CU_TRY(key_out.alloc(size_t(n) * r.gwidth + 16, s));
    CU_TRY(t_out.alloc(size_t(n) * 8 + 16, s));
    CU_TRY(v_out.alloc(size_t(n) * 8 + 16, s));
    if (n > 0)
      k::range_fn_gather(L, fv.idx.as<uint32_t>(), d_n, n, ColView{r.gkey.p, nullptr, gtype, r.gwidth, nullptr}, r.win_t.as<int64_t>(),
                         fv.value.as<double>(), key_out.p, t_out.as<int64_t>(), v_out.as<double>());
    std::vector<ExportCol> srcs{{col_name(c.schema, uint32_t(c.agg->group_col)), gtype, key_out.p, r.gwidth, false}, {"t", T_I64, t_out.p, 8, false},
                                {"value", T_F64, v_out.p, 8, false}};
    return export_groups(e, srcs, n, nullptr, r.ag.st.d2h, out);
  }

  RangeFnSums sums;
  int rc = range_fn_sums(e, c, &fv, &sums);
  if (!rc) rc = read_counts(e, hn, d_n, sizeof(hn));
  if (rc) return rc;
  const AggBuffers& ab = sums.ab;
  std::vector<ExportCol> srcs{{"group", T_U32, ab.gkey.p, 4, false}, {"t", T_I64, ab.bucket.p, 8, false}, {"count", T_U64, ab.count.p, 8, false},
                              {"sum", T_F64, ab.sum.p, 8, false},    {"min", T_F64, ab.mn.p, 8, false},    {"max", T_F64, ab.mx.p, 8, false}};
  return export_groups(e, srcs, hn[1], nullptr, r.ag.st.d2h, out);
}

// hg_scan_range_function and its by-map form
static int range_function_entry(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                                size_t n_preds, const hg_agg_spec* agg, const hg_range_spec* range, uint32_t fn, const hg_group_map* map,
                                struct ArrowArrayStream* out) {
  AggCall c;
  int rc = prepare_call(&c, schema, ssts, n_ssts, agg);
  if (!rc) rc = prepare_range(&c, preds, n_preds, range, fn, map);
  if (rc) return rc;
  return range_fn_call(e, c, [&](RangeFnValues& fv) { return range_function_tail(e, c, fv, out); });
}

int hg_scan_range_function(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                           size_t n_preds, const hg_agg_spec* agg, const hg_range_spec* range, uint32_t fn, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  return range_function_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, range, fn, nullptr, out);
  HG_GUARD_END
}

int hg_scan_range_function_by_map(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                                  size_t n_preds, const hg_agg_spec* agg, const hg_range_spec* range, uint32_t fn, const hg_group_map* map,
                                  struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  if (!map) return set_error(HG_ERR_INVALID, "null group map");
  return range_function_entry(e, schema, ssts, n_ssts, preds, n_preds, agg, range, fn, map, out);
  HG_GUARD_END
}

// ------------------------------------------------------------------------------------------------- top-k / bottom-k by label group
// The windows with a value (range_fn_values), ranked: one stable 64-bit radix_sort_pairs of idx by the rank key of the value, then
// range_fn_segments with the by-map call's key (ordinal << shift) | j, so that each (group, t) run is in (rank key, series) order; the
// first k windows of each run are kept (topk_keep + compact_flags: cnt[2] rows) and gathered with their series key.
static int range_topk_tail(hg_engine* e, const AggCall& c, RangeFnValues& fv, uint32_t topk, uint32_t order, struct ArrowArrayStream* out) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const RangeState& r = fv.r;
  const uint32_t W = fv.W;
  uint32_t* d_n = fv.d_n();
  if (W > 0) {
    // the windows in (series, t) order, stably by value: equal rank keys keep their series order
    DevBuf keys, keys2, idx2, rcounts;
    CU_TRY(keys.alloc(size_t(W) * 8 + 16, s));
    CU_TRY(keys2.alloc(size_t(W) * 8 + 16, s));
    CU_TRY(idx2.alloc(size_t(W) * 4 + 16, s));
    CU_TRY(rcounts.alloc(k::radix_tmp_elems(W) * sizeof(uint32_t), s));
    k::topk_rank_keys(L, fv.idx.as<uint32_t>(), d_n, W, fv.value.as<double>(), order == HG_TOPK, keys.as<uint64_t>());
    if (k::radix_sort_pairs(L, keys.as<uint64_t>(), fv.idx.as<uint32_t>(), keys2.as<uint64_t>(), idx2.as<uint32_t>(), d_n, W, 64,
                            rcounts.as<uint32_t>()))
      std::swap(fv.idx, idx2);
  }
  RangeFnSegments sg;
  int rc = range_fn_segments(e, c, &fv, &sg);
  if (rc) return rc;
  DevBuf keep, pos;
  CU_TRY(keep.alloc(size_t(W) + 16, s));
  CU_TRY(pos.alloc(size_t(W) * 4 + 16, s));
  k::topk_keep(L, sg.seg.as<uint32_t>(), d_n, W, topk, keep.as<uint8_t>());
  if (W > 0) k::compact_flags(L, keep.as<uint8_t>(), W, fv.ctmp.as<uint32_t>(), pos.as<uint32_t>(), d_n + 2);
  uint32_t hn[3] = {0, 0, 0};
  rc = read_counts(e, hn, d_n, sizeof(hn));
  if (rc) return rc;
  const uint32_t n = hn[2], gtype = c.schema->types[c.agg->group_col], kw = type_width(gtype);
  DevBuf g_out, t_out, key_out, v_out;
  CU_TRY(g_out.alloc(size_t(n) * 4 + 16, s));
  CU_TRY(t_out.alloc(size_t(n) * 8 + 16, s));
  CU_TRY(key_out.alloc(size_t(n) * kw + 16, s));
  CU_TRY(v_out.alloc(size_t(n) * 8 + 16, s));
  k::topk_gather(L, pos.as<uint32_t>(), d_n + 2, n, sg.vals.as<uint32_t>(), r.gkey.as<uint32_t>(), r.win_t.as<int64_t>(), fv.value.as<double>(),
                 r.win_lo.as<uint32_t>(), r.ag.spec.group, r.ag.rows,
                 k::TopkOut{g_out.as<uint32_t>(), t_out.as<int64_t>(), key_out.p, v_out.as<double>()});
  std::vector<ExportCol> srcs{{"group", T_U32, g_out.p, 4, false}, {"t", T_I64, t_out.p, 8, false},
                              {col_name(c.schema, uint32_t(c.agg->group_col)), gtype, key_out.p, kw, false}, {"value", T_F64, v_out.p, 8, false}};
  return export_groups(e, srcs, n, nullptr, r.ag.st.d2h, out);
}

int hg_scan_range_function_topk(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                                size_t n_preds, const hg_agg_spec* agg, const hg_range_spec* range, uint32_t fn, const hg_group_map* map, uint32_t k,
                                uint32_t order, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  if (!map) return set_error(HG_ERR_INVALID, "null group map");
  // the by-map range function call's preparation, with k and the order checked before the map is read
  AggCall c;
  int rc = prepare_call(&c, schema, ssts, n_ssts, agg);
  if (!rc) rc = prepare_range(&c, preds, n_preds, range, fn, map, [&](const hg_group_map**) -> int {
    if (k == 0) return set_error(HG_ERR_INVALID, "top-k: k must be >= 1");
    if (order != HG_TOPK && order != HG_BOTTOMK) return set_error(HG_ERR_INVALID, "top-k: order is not an hg_topk_order");
    return HG_OK;
  });
  if (rc) return rc;
  return range_fn_call(e, c, [&](RangeFnValues& fv) { return range_topk_tail(e, c, fv, k, order, out); });
  HG_GUARD_END
}

// ------------------------------------------------------------------------------------------------- histogram quantiles
// A histogram map made dense on the host: the map's distinct groups and distinct upper bounds sorted once (ranks), and every key's
// (group rank, bound rank) pair as one internal u32 ordinal, the index of the pair among the map's distinct pairs.  The windows carry that
// ordinal through range_stage as the by-map call's windows carry the caller's.
struct HistogramMap {
  std::vector<uint32_t> ordinal;            // per map entry
  std::vector<k::BucketPair> pair;          // ordinal -> (group rank, bound rank)
  std::vector<double> bounds;               // bound rank -> upper bound, ascending (-0.0 taken as +0.0)
  std::vector<uint32_t> groups;             // group rank -> the caller's ordinal, ascending
  int gbits = 0, lbits = 0;                 // the bits of the largest group rank and bound rank
};

static int prepare_histogram_map(const hg_group_map* map, const double* upper_bounds, HistogramMap* hm) {
  const uint32_t n = map->count;
  if (n && !upper_bounds) return set_error(HG_ERR_INVALID, "histogram map: null upper bounds");
  for (uint32_t i = 0; i < n; i++)
    if (upper_bounds[i] != upper_bounds[i]) return set_error(HG_ERR_INVALID, "histogram map: a NaN upper bound");
  auto distinct = [](auto v) { std::sort(v.begin(), v.end()); v.erase(std::unique(v.begin(), v.end()), v.end()); return v; };
  std::vector<double> b(upper_bounds, upper_bounds + n);
  for (double& x : b) x = x + 0.0;          // -0.0 + 0.0 = +0.0: one bound, one representation
  hm->groups = distinct(std::vector<uint32_t>(map->groups, map->groups + n));
  hm->bounds = distinct(b);
  auto rank = [](const auto& v, auto x) { return uint32_t(std::lower_bound(v.begin(), v.end(), x) - v.begin()); };
  std::vector<uint64_t> p(n);
  for (uint32_t i = 0; i < n; i++) p[i] = (uint64_t(rank(hm->groups, map->groups[i])) << 32) | rank(hm->bounds, b[i]);
  const std::vector<uint64_t> pairs = distinct(p);
  hm->pair.resize(pairs.size());
  for (size_t j = 0; j < pairs.size(); j++) hm->pair[j] = k::BucketPair{uint32_t(pairs[j] >> 32), uint32_t(pairs[j])};
  hm->ordinal.resize(n);
  for (uint32_t i = 0; i < n; i++) hm->ordinal[i] = rank(pairs, p[i]);
  hm->gbits = bit_length(hm->groups.empty() ? 0 : hm->groups.size() - 1);
  hm->lbits = bit_length(hm->bounds.empty() ? 0 : hm->bounds.size() - 1);
  return HG_OK;
}

// The windows with a value (range_fn_values over the internal ordinals), their sums per (group, t, bound) (range_fn_sums with the key
// (group rank, step, bound rank)), those sums cut into (group, t) segments, and bucketQuantile per segment
static int histogram_quantile_tail(hg_engine* e, const AggCall& c, RangeFnValues& fv, const HistogramMap& hm, const double* quantiles,
                                   uint32_t n_quantiles, struct ArrowArrayStream* out) {
  cudaStream_t s = e->stream;
  Launch L = e->L();
  const uint32_t W = fv.W;
  uint32_t* d_n = fv.d_n();
  // the tables of the dense map go up once, when there are windows to read them
  DevBuf pair, bounds, groups;
  if (W > 0) {
    const size_t pb = hm.pair.size() * sizeof(k::BucketPair), bb = hm.bounds.size() * 8, gb = hm.groups.size() * 4;
    CU_TRY(pair.alloc(pb + 16, s));
    CU_TRY(bounds.alloc(bb + 16, s));
    CU_TRY(groups.alloc(gb + 16, s));
    CU_TRY(cudaMemcpyAsync(pair.p, hm.pair.data(), pb, cudaMemcpyHostToDevice, s));
    CU_TRY(cudaMemcpyAsync(bounds.p, hm.bounds.data(), bb, cudaMemcpyHostToDevice, s));
    CU_TRY(cudaMemcpyAsync(groups.p, hm.groups.data(), gb, cudaMemcpyHostToDevice, s));
    e->stats.bytes_h2d += pb + bb + gb;
  }
  RangeFnSums sums;
  int rc = range_fn_sums(e, c, &fv, &sums, hm.gbits + c.shift + hm.lbits, [&](uint64_t* keys, uint32_t* vals) {
    k::histogram_sort_keys(L, fv.idx.as<uint32_t>(), d_n, W, fv.r.gkey.as<uint32_t>(), pair.as<k::BucketPair>(), fv.r.win_t.as<int64_t>(), c.rs.start,
                           c.rs.step, c.shift, hm.lbits, keys, vals);
  });
  if (rc) return rc;
  AggBuffers& ab = sums.ab;
  DevBuf seg;
  CU_TRY(seg.alloc(size_t(W) * 4 + 16, s));
  if (W > 0) {
    // the sums in (group, t, bound) order cut again where (group, t) changes: cnt[2] segments
    k::histogram_heads(L, ab.gkey.as<uint32_t>(), ab.bucket.as<int64_t>(), pair.as<k::BucketPair>(), d_n + 1, W, sums.head.as<uint8_t>());
    k::clear_tail(L, sums.head.as<uint8_t>(), d_n + 1, W);
    k::compact_flags(L, sums.head.as<uint8_t>(), W, fv.ctmp.as<uint32_t>(), seg.as<uint32_t>(), d_n + 2);
  }
  uint32_t hn[3] = {0, 0, 0};
  rc = read_counts(e, hn, d_n, sizeof(hn));
  if (rc) return rc;
  const uint32_t S = hn[2];
  DevBuf g_out, t_out, forced, qout;
  CU_TRY(g_out.alloc(size_t(S) * 4 + 16, s));
  CU_TRY(t_out.alloc(size_t(S) * 8 + 16, s));
  CU_TRY(forced.alloc(size_t(S) + 16, s));
  CU_TRY(qout.alloc(size_t(S) * n_quantiles * 8 + 16, s));
  k::histogram_quantile(L, quantile_spec(quantiles, n_quantiles), seg.as<uint32_t>(), S, hn[1], ab.gkey.as<uint32_t>(), ab.bucket.as<int64_t>(),
                        ab.sum.as<double>(), pair.as<k::BucketPair>(), bounds.as<double>(), groups.as<uint32_t>(),
                        k::HistogramOut{g_out.as<uint32_t>(), t_out.as<int64_t>(), forced.as<uint8_t>(), qout.as<double>()});
  std::vector<ExportCol> srcs{{"group", T_U32, g_out.p, 4, false}, {"t", T_I64, t_out.p, 8, false}, {"forced_monotonic", T_U8, forced.p, 1, false}};
  for (uint32_t j = 0; j < n_quantiles; j++) srcs.push_back({"quantile_" + std::to_string(j), T_F64, qout.as<double>() + size_t(j) * S, 8, false});
  return export_groups(e, srcs, S, nullptr, fv.r.ag.st.d2h, out);
}

int hg_scan_histogram_quantile(hg_engine* e, const hg_schema_desc* schema, const hg_sst_desc* ssts, size_t n_ssts, const hg_predicate* preds,
                               size_t n_preds, const hg_agg_spec* agg, const hg_range_spec* range, uint32_t fn, const hg_group_map* map,
                               const double* upper_bounds, const double* quantiles, uint32_t n_quantiles, struct ArrowArrayStream* out) {
  HG_GUARD_BEGIN
  if (!e || !out) return set_error(HG_ERR_INVALID, "null argument");
  if (!map) return set_error(HG_ERR_INVALID, "null group map");
  // the by-map range function call's preparation; before the map is read, the quantile list, the bounds and the dense map, which is
  // the map prepared (a key with two different (group, bound) pairs has two internal ordinals: prepare_by_map refuses it); then the
  // width of the sort key
  HistogramMap hm;
  hg_group_map dense{};
  AggCall c;
  int rc = prepare_call(&c, schema, ssts, n_ssts, agg);
  if (!rc) rc = prepare_range(&c, preds, n_preds, range, fn, map, [&](const hg_group_map** m) -> int {
    int rc = check_quantile_spec(schema, agg, quantiles, n_quantiles);
    if (!rc) rc = prepare_histogram_map(*m, upper_bounds, &hm);
    if (rc) return rc;
    dense = hg_group_map{(*m)->keys, hm.ordinal.data(), (*m)->count, 0};
    *m = &dense;
    return HG_OK;
  });
  if (rc) return rc;
  if (hm.gbits + c.shift + hm.lbits > 64)
    return set_error(HG_ERR_UNSUPPORTED, "histogram quantile: the sort key (group, step, bound) needs more than 64 bits");
  return range_fn_call(e, c, [&](RangeFnValues& fv) { return histogram_quantile_tail(e, c, fv, hm, quantiles, n_quantiles, out); });
  HG_GUARD_END
}

}  // extern "C"
