// chunk_scratch.h — the layout of a column chunk's decode scratch in the general pipeline.  parquet_meta.cpp sizes every chunk with
// these functions, and the kernels that fill and read the scratch (snappy_pages_kernel, zstd_chunks_kernel, decode_chunks_kernel)
// walk it with the same ones, so the host and the device cannot disagree about where a chunk's bytes are.
//
// A row group's scratch holds its selected chunks back to back in ColSel order (chunk_scratch_off).  One chunk's scratch is, in order:
//   1. the decompressed dictionary page (compressed chunks with a dictionary page);
//   2. the BYTE_ARRAY dictionary's entry table (byte_dict_table_bytes);
//   3. per data page: the decompressed page (compressed chunks), then the page's PLAIN image or its length / index run
//      (page_has_image: DELTA and dictionary pages);
//   4. the Zstandard literal buffer (Zstandard chunks).
// Every part is one region: its bytes rounded up to 16, plus 32 bytes of slack.  The page functions take PageDev (device) or PageMeta
// (host); both have the same field names.
#pragma once
#include "device_types.h"

namespace horae {

// Zstandard's largest block (zst::kBlockMax): no block has more literals, so the literal buffer never needs more
constexpr uint32_t kZstdLitMax = 128u << 10;

HORAE_HD uint64_t scratch_region(uint64_t bytes) { return (bytes + 15) / 16 * 16 + 32; }

// 1 + 2: what precedes the first data page.  dict_uncomp == 0: the chunk has no dictionary page.
HORAE_HD uint64_t dict_body_scratch(uint32_t codec, uint32_t dict_uncomp) {
  return dict_uncomp && codec != CODEC_UNCOMPRESSED ? scratch_region(dict_uncomp) : 0;
}
// The entry table of a BYTE_ARRAY dictionary: one (offset in the page, length) u32 pair per entry.  Every entry takes at least its
// 4-byte length, so dict_uncomp / 4 bounds the entry count and the table's size follows from the page size alone.
HORAE_HD uint64_t byte_dict_table_bytes(uint32_t dict_uncomp) { return scratch_region(uint64_t(dict_uncomp) / 4 * 8); }
HORAE_HD uint64_t dict_scratch(uint32_t codec, uint32_t phys, uint32_t dict_uncomp) {
  return dict_body_scratch(codec, dict_uncomp) + (dict_uncomp && phys == PT_BYTE_ARRAY ? byte_dict_table_bytes(dict_uncomp) : 0);
}

// 3: one data page.  decode_chunks_kernel expands these encodings into 8 bytes per value (at most) before it reads them.
HORAE_HD bool page_has_image(uint32_t encoding) {
  return encoding == ENC_DELTA_BINARY_PACKED || encoding == ENC_DELTA_LENGTH_BYTE_ARRAY || encoding == ENC_DELTA_BYTE_ARRAY ||
         encoding == ENC_RLE_DICT || encoding == ENC_PLAIN_DICT;
}
template <class Page> HORAE_HD uint64_t page_body_scratch(uint32_t codec, const Page& pg) {
  return codec != CODEC_UNCOMPRESSED ? scratch_region(pg.uncomp_size) : 0;
}
template <class Page> HORAE_HD uint64_t page_image_scratch(const Page& pg) {
  return page_has_image(pg.encoding) ? scratch_region(uint64_t(pg.num_values) * 8) : 0;
}

// 4: the literal buffer of a Zstandard chunk, sized by the chunk's largest page (dictionary page included) and capped at kZstdLitMax.
template <class Page> HORAE_HD uint64_t zstd_lit_scratch(uint32_t dict_uncomp, const Page* pages, uint32_t npages) {
  uint32_t big = dict_uncomp;
  for (uint32_t p = 0; p < npages; p++) { const uint32_t u = pages[p].uncomp_size; big = u > big ? u : big; }
  return scratch_region(big < kZstdLitMax ? big : kZstdLitMax);
}

// The whole chunk: ChunkDev::scratch_bytes.
template <class Page>
HORAE_HD uint64_t chunk_scratch_bytes(uint32_t codec, uint32_t phys, uint32_t dict_uncomp, const Page* pages, uint32_t npages) {
  uint64_t n = dict_scratch(codec, phys, dict_uncomp);
  for (uint32_t p = 0; p < npages; p++) n += page_body_scratch(codec, pages[p]) + page_image_scratch(pages[p]);
  if (codec == CODEC_ZSTD) n += zstd_lit_scratch(dict_uncomp, pages, npages);
  return n;
}

// Base of selected column ci's chunk inside its row group's scratch.
HORAE_HD uint64_t chunk_scratch_off(const RgSel& rs, const ChunkDev* chunks, const ColSel* cols, int ci) {
  uint64_t off = rs.scratch_off;
  for (int j = 0; j < ci; j++) off += chunks[cols[j].col].scratch_bytes;      // 0 for uncompressed chunks without DELTA / dictionary pages
  return off;
}

// Where a data page's compressed stream lies in its payload and how long its decompressed output is.  A V2 page keeps its levels
// uncompressed in front of the stream, and its values are compressed only if v2_compressed says so.
struct PageStream {
  uint32_t skip;       // payload bytes before the stream
  uint32_t comp;       // bytes of the stream
  uint32_t out;        // bytes it decompresses to
  bool compressed;
};
template <class Page> HORAE_HD PageStream page_stream(const Page& pg) {
  const uint32_t skip = pg.page_type == PAGE_DATA_V2 ? pg.v2_def_len + pg.v2_rep_len : 0u;
  return PageStream{skip, pg.comp_size - skip, pg.uncomp_size - skip, pg.page_type != PAGE_DATA_V2 || pg.v2_compressed != 0};
}

}  // namespace horae
