// parquet_meta.cpp — see parquet_meta.hpp.
#include "parquet_meta.hpp"
#include "chunk_scratch.h"

#include <algorithm>


namespace horae {
namespace {

// Thrift compact protocol reader (field-id deltas, zigzag varints, nested skip).
class Compact {
 public:
  Compact(const uint8_t* p, const uint8_t* end) : p_(p), end_(end) {}
  bool ok() const { return ok_; }
  const uint8_t* pos() const { return p_; }

  uint64_t uvar() {
    uint64_t v = 0;
    for (int shift = 0; shift < 64; shift += 7) {
      if (p_ >= end_) return fail();
      uint8_t b = *p_++;
      v |= uint64_t(b & 0x7f) << shift;
      if (!(b & 0x80)) return v;
    }
    return fail();
  }
  int64_t svar() {
    uint64_t v = uvar();
    return int64_t(v >> 1) ^ -int64_t(v & 1);
  }
  // Iterates the fields of a struct: cb(field_id, wire_type) must consume the value (or call skip).
  template <class F>
  void each_field(F&& cb) {
    // nesting cap: footers / page headers are untrusted bytes and skip() recurses through structs, lists and maps
    if (++depth_ > kMaxDepth) { fail(); --depth_; return; }
    struct Leave { int& d; ~Leave() { --d; } } leave{depth_};
    int fid = 0;
    while (ok_) {
      if (p_ >= end_) { fail(); return; }
      uint8_t h = *p_++;
      if (h == 0) return;
      int wt = h & 0x0f, delta = h >> 4;
      fid = delta ? fid + delta : int(svar());
      cb(fid, wt);
    }
  }
  // Iterates list elements: cb(index, elem_wire_type)
  template <class F>
  void each_elem(F&& cb) {
    if (++depth_ > kMaxDepth) { fail(); --depth_; return; }
    struct Leave { int& d; ~Leave() { --d; } } leave{depth_};
    if (p_ >= end_) { fail(); return; }
    uint8_t h = *p_++;
    uint64_t n = h >> 4;
    int et = h & 0x0f;
    if (n == 15) n = uvar();
    for (uint64_t i = 0; i < n && ok_; i++) cb(int(i), et);
  }
  std::string str() {
    uint64_t n = uvar();
    if (!ok_ || uint64_t(end_ - p_) < n) { fail(); return {}; }
    std::string s(reinterpret_cast<const char*>(p_), n);
    p_ += n;
    return s;
  }
  // a binary field, left in place: *v = its first byte, *n = its length
  bool binary(const uint8_t** v, uint64_t* n) {
    *n = uvar();
    if (!ok_ || uint64_t(end_ - p_) < *n) { fail(); return false; }
    *v = p_;
    p_ += *n;
    return true;
  }
  void skip(int wt) {
    switch (wt) {
      case 1: case 2: return;  // bool lives in the field header
      case 3: advance(1); return;
      case 4: case 5: case 6: (void)uvar(); return;
      case 7: advance(8); return;
      case 8: { uint64_t n = uvar(); advance(n); return; }
      case 9: case 10:
        each_elem([&](int, int et) { if (et == 1 || et == 2) advance(1); else skip(et); });
        return;
      case 11: {
        uint64_t n = uvar();
        if (n == 0) return;
        if (p_ >= end_) { fail(); return; }
        uint8_t kv = *p_++;
        if (++depth_ > kMaxDepth) { fail(); --depth_; return; }
        for (uint64_t i = 0; i < n && ok_; i++) { skip(kv >> 4); skip(kv & 0x0f); }
        --depth_;
        return;
      }
      case 12: each_field([&](int, int t) { skip(t); }); return;
      default: fail();
    }
  }

 private:
  uint64_t fail() { ok_ = false; return 0; }
  void advance(uint64_t n) { if (uint64_t(end_ - p_) < n) fail(); else p_ += n; }
  static constexpr int kMaxDepth = 32;
  const uint8_t* p_;
  const uint8_t* end_;
  bool ok_ = true;
  int depth_ = 0;
};

// max_value (5) / min_value (6): values of 1 to 8 bytes into max / min; with `arena` (BYTE_ARRAY chunks) every value, whole, into it
void read_stats(Compact& c, ColumnStats* st, std::vector<uint8_t>* arena) {
  auto bound = [&](uint8_t dst[8], bool* has, bool* has_bin, uint32_t* off, uint32_t* len) {
    const uint8_t* v = nullptr;
    uint64_t n = 0;
    if (!c.binary(&v, &n)) return;
    *has = n > 0 && n <= 8;
    if (*has) { std::memset(dst, 0, 8); std::memcpy(dst, v, n); }
    if (arena) {
      *has_bin = true;
      *off = uint32_t(arena->size());
      *len = uint32_t(n);
      arena->insert(arena->end(), v, v + n);
    }
  };
  c.each_field([&](int fid, int wt) {
    if (fid == 5 && wt == 8) bound(st->max, &st->has_max, &st->has_bin_max, &st->bin_max_off, &st->bin_max_len);
    else if (fid == 6 && wt == 8) bound(st->min, &st->has_min, &st->has_bin_min, &st->bin_min_off, &st->bin_min_len);
    else if (fid == 3 && wt == 6) { st->null_count = c.svar(); st->has_null_count = true; }
    else c.skip(wt);
  });
}

void read_column_meta(Compact& c, ChunkMeta* cm, std::vector<uint8_t>* stat_bytes) {
  c.each_field([&](int fid, int wt) {
    switch (fid) {
      case 1: cm->phys_type = int(c.svar()); break;
      case 4: cm->codec = int(c.svar()); break;
      case 5: cm->num_values = c.svar(); break;
      case 7: cm->total_compressed = c.svar(); break;
      case 9: cm->data_page_offset = c.svar(); break;
      case 11: cm->dict_page_offset = c.svar(); break;
      // (writers put type (1) before statistics (12), as parquet.thrift numbers them; a footer that does not keeps no Binary bounds)
      case 12: read_stats(c, &cm->stats, cm->phys_type == PT_BYTE_ARRAY ? stat_bytes : nullptr); break;
      case 14: if (wt == 6) cm->bloom_offset = c.svar(); else c.skip(wt); break;
      case 15: if (wt == 5) { cm->bloom_length = int32_t(c.svar()); cm->has_bloom_length = true; } else c.skip(wt); break;
      default: c.skip(wt);
    }
  });
}

struct PageHeader {
  int type = 0;
  int32_t uncomp = 0, comp = 0;
  int32_t num_values = 0, encoding = 0, def_level_encoding = 3;   // (RLE; V2 pages have no other)
  int32_t v2_def_len = 0, v2_rep_len = 0;
  bool v2_compressed = true;
  size_t header_len = 0;
};

bool read_page_header(const uint8_t* p, const uint8_t* end, PageHeader* h) {
  Compact c(p, end);
  c.each_field([&](int fid, int wt) {
    if (fid == 1) h->type = int(c.svar());
    else if (fid == 2) h->uncomp = int32_t(c.svar());
    else if (fid == 3) h->comp = int32_t(c.svar());
    else if (fid == 5 && wt == 12) {
      c.each_field([&](int f2, int t2) {
        if (f2 == 1) h->num_values = int32_t(c.svar());
        else if (f2 == 2) h->encoding = int32_t(c.svar());
        else if (f2 == 3) h->def_level_encoding = int32_t(c.svar());
        else c.skip(t2);
      });
    } else if (fid == 7 && wt == 12) {      // DictionaryPageHeader
      c.each_field([&](int f2, int t2) {
        if (f2 == 1) h->num_values = int32_t(c.svar());
        else if (f2 == 2) h->encoding = int32_t(c.svar());
        else c.skip(t2);
      });
    } else if (fid == 8 && wt == 12) {
      c.each_field([&](int f2, int t2) {
        if (f2 == 1) h->num_values = int32_t(c.svar());
        else if (f2 == 4) h->encoding = int32_t(c.svar());
        else if (f2 == 5) h->v2_def_len = int32_t(c.svar());
        else if (f2 == 6) h->v2_rep_len = int32_t(c.svar());
        else if (f2 == 7) h->v2_compressed = (t2 == 1);
        else c.skip(t2);
      });
    } else c.skip(wt);
  });
  h->header_len = size_t(c.pos() - p);
  if (h->uncomp < 0 || h->comp < 0 || h->num_values < 0 || h->v2_def_len < 0 || h->v2_rep_len < 0) return false;   // sizes are i32 on the wire
  return c.ok();
}

}  // namespace

bool bloom_bitset(const uint8_t* data, size_t len, const ChunkMeta& cm, uint64_t* bitset_off, uint32_t* num_bytes) {
  if (cm.phys_type == PT_BYTE_ARRAY || cm.bloom_offset < 4 || len < 12 || uint64_t(cm.bloom_offset) >= len - 8) return false;
  if (cm.has_bloom_length && cm.bloom_length < 0) return false;
  uint64_t end = len - 8;                                 // the footer length and the magic are never part of a filter
  if (cm.has_bloom_length) end = std::min<uint64_t>(end, uint64_t(cm.bloom_offset) + uint64_t(cm.bloom_length));
  Compact c(data + cm.bloom_offset, data + end);
  int64_t nbytes = -1;
  int unions = 0;                                         // bit k: union field 2 + k holds exactly its known member (field 1)
  c.each_field([&](int fid, int wt) {
    if (fid == 1 && wt == 5) nbytes = c.svar();
    else if (fid >= 2 && fid <= 4 && wt == 12) {
      bool known = false, other = false;
      c.each_field([&](int f2, int t2) { if (f2 == 1 && t2 == 12) known = true; else other = true; c.skip(t2); });
      if (known && !other) unions |= 1 << (fid - 2);
    } else c.skip(wt);
  });
  if (!c.ok() || unions != 7 || nbytes < 32 || nbytes > (int64_t(128) << 20) || (nbytes & (nbytes - 1)) != 0) return false;
  const uint64_t off = uint64_t(c.pos() - data);
  if (off + uint64_t(nbytes) > end) return false;
  *bitset_off = off;
  *num_bytes = uint32_t(nbytes);
  return true;
}

bool parse_parquet(const uint8_t* data, size_t len, FileMetaData* out, std::string* err) {
  auto bad = [&](const char* m) { if (err) *err = m; return false; };
  if (len < 12 || std::memcmp(data, "PAR1", 4) != 0 || std::memcmp(data + len - 4, "PAR1", 4) != 0)
    return bad("not a Parquet file (magic)");
  uint32_t mlen;
  std::memcpy(&mlen, data + len - 8, 4);
  if (uint64_t(mlen) + 12 > len) return bad("footer length out of range");
  *out = FileMetaData();
  Compact c(data + len - 8 - mlen, data + len - 8);
  c.each_field([&](int fid, int wt) {
    if (fid == 2 && wt == 9) {
      c.each_elem([&](int idx, int) {
        int rep = 0, type = -1, nchildren = 0;
        std::string name;
        c.each_field([&](int f2, int t2) {
          if (f2 == 1) type = int(c.svar());
          else if (f2 == 3) rep = int(c.svar());
          else if (f2 == 4) name = c.str();
          else if (f2 == 5) nchildren = int(c.svar());
          else c.skip(t2);
        });
        if (idx > 0) {
          (void)nchildren;
          out->repetition.push_back(rep);
          out->phys_types.push_back(type);
          out->names.push_back(name);
        }
      });
      out->ncols = int(out->names.size());
    } else if (fid == 3 && wt == 6) {
      out->num_rows = c.svar();
    } else if (fid == 4 && wt == 9) {
      c.each_elem([&](int, int) {
        RowGroupMeta rg;
        c.each_field([&](int f2, int t2) {
          if (f2 == 1 && t2 == 9) {
            c.each_elem([&](int, int) {
              ChunkMeta cm;
              c.each_field([&](int f3, int t3) {
                if (f3 == 3 && t3 == 12) read_column_meta(c, &cm, &out->stat_bytes);
                else c.skip(t3);
              });
              rg.cols.push_back(cm);
            });
          } else if (f2 == 3 && t2 == 6) {
            rg.num_rows = c.svar();
          } else c.skip(t2);
        });
        out->rgs.push_back(std::move(rg));
      });
    } else c.skip(wt);
  });
  if (!c.ok()) return bad("thrift error in footer");

  // Walk the data pages of every chunk (page counts come from the headers, never assumed: SURVEY §8 caveat).
  int64_t row = 0;
  size_t rgi = 0;
  for (auto& rg : out->rgs) {
    if (int(rg.cols.size()) != out->ncols) return bad("row group column count mismatch");
    // page headers sit tens of KB apart (one cache miss each, on pinned host memory): ask for the headers of the row group after next
    if (rgi + 2 < out->rgs.size())
      for (const auto& nc : out->rgs[rgi + 2].cols) {
        const int64_t o = (nc.dict_page_offset > 0 && nc.dict_page_offset < nc.data_page_offset) ? nc.dict_page_offset : nc.data_page_offset;
        if (o >= 0 && uint64_t(o) + 64 <= len) { __builtin_prefetch(data + o); __builtin_prefetch(data + o + 63); }
      }
    rgi++;
    rg.first_row = row;
    row += rg.num_rows;
    for (auto& cm : rg.cols) {
      cm.first_page = uint32_t(out->pages.size());
      uint64_t pos = uint64_t(cm.data_page_offset);
      if (cm.dict_page_offset > 0 && cm.dict_page_offset < cm.data_page_offset) pos = uint64_t(cm.dict_page_offset);   // dictionary page first
      int64_t seen = 0;
      while (seen < cm.num_values) {
        if (pos >= len) return bad("page offset beyond end of file");
        PageHeader h;
        if (!read_page_header(data + pos, data + len, &h)) return bad("thrift error in page header");
        uint64_t payload = pos + h.header_len;
        if (h.comp < 0 || payload + uint64_t(h.comp) > len) return bad("page payload beyond end of file");
        pos = payload + uint64_t(h.comp);
        if (h.type == PAGE_DICT) {
          cm.has_dict_page = true;
          cm.dict_payload_off = payload;
          cm.dict_comp_size = uint32_t(h.comp);
          cm.dict_uncomp_size = uint32_t(h.uncomp);
          cm.dict_num_values = uint32_t(h.num_values);
          continue;
        }
        if (h.type != PAGE_DATA && h.type != PAGE_DATA_V2) continue;
        PageMeta pm;
        pm.payload_off = payload;
        pm.comp_size = uint32_t(h.comp);
        pm.uncomp_size = uint32_t(h.uncomp);
        pm.num_values = uint32_t(h.num_values);
        pm.page_type = uint8_t(h.type);
        pm.encoding = uint8_t(h.encoding);
        pm.def_level_encoding = uint8_t(h.def_level_encoding);
        pm.v2_def_len = uint32_t(h.v2_def_len);
        pm.v2_rep_len = uint32_t(h.v2_rep_len);
        pm.v2_compressed = h.v2_compressed ? 1 : 0;
        out->pages.push_back(pm);
        seen += h.num_values;
        if (h.num_values <= 0) return bad("page with no values");
      }
      if (seen != cm.num_values) return bad("page value counts do not add up to the chunk");
      cm.num_pages = uint32_t(out->pages.size()) - cm.first_page;
      cm.scratch_bytes = chunk_scratch_bytes(uint32_t(cm.codec), uint32_t(cm.phys_type), cm.has_dict_page ? cm.dict_uncomp_size : 0u,
                                             out->pages.data() + cm.first_page, cm.num_pages);
    }
  }
  return true;
}

}  // namespace horae
