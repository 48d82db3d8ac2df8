/*
 * horae_oracle.c — CPU ORACLE for the columnar hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This file is the parity checker and the "port" CPU baseline.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load it.  The product (horaedb_b200/csrc) never links,
 * imports or calls anything in oracle/.
 *
 * It restates, in plain C, the reference's scan / compaction pipeline (all citations relative to
 * /root/reference, apache/horaedb @ 9cec5636):
 *
 *   S1/S2  Parquet decode of the SST format fixed by build_write_props (src/columnar_storage/src/storage.rs:258-298)
 *          and WriteConfig::default (config.rs:120-133).  The arithmetic lives in the un-vendored crates
 *          parquet 53.2.0 / snap 1.1.1 (Cargo.lock:2454, 3145); restated here from the published Apache Parquet
 *          format spec (Thrift compact footer + page headers, RLE/bit-packed hybrid levels, PLAIN values) and the
 *          Snappy raw-block format; Zstandard pages (ParquetCompression::Zstd, config.rs:78-94; zstd 0.13.2, Cargo.lock:3893) through
 *          zstd_oracle.h, a sequential restatement of RFC 8878.  Pinned in tests against pyarrow 24 (independent C++ implementation;
 *          its codecs are libsnappy / libzstd themselves).
 *   S2     row-group pruning = DataFusion PruningPredicate as pinned by the plan text at read.rs:613
 *          ("CASE WHEN null_count = row_count THEN false ELSE min <= lit AND lit <= max").
 *   S3     FilterExec(conjunction(predicates)) BEFORE the merge (read.rs:459-470); NULL => false.
 *   S4     SortPreservingMergeExec on (pk0..pkN-1 ASC NULLS FIRST, __seq__ ASC) (read.rs:412-427, 479-480),
 *          ties -> lower stream index; output re-batched at batch_size (datafusion 43 default 8192); a single
 *          input partition is passed through un-rebatched.
 *   S5     MergeStream::merge_batch / primary_key_eq / poll_next (read.rs:262-384): PK-run grouping, pending carry
 *          across batches, one output batch per input batch (None when empty), final flush of pending.
 *   S6     LastValueOperator::merge (operator.rs:39-44): last row of the run.
 *   S8/A1  Timestamp::truncate_by (types.rs:82-85): truncating i64 division.
 *   A2     aggregation over post-dedup rows (absent in the reference; SURVEY §8a A1-A3): count(*) u64,
 *          sum f64 by SEQUENTIAL addition in stream order, min/max by < / >.   PARITY UNPINNED by the reference.
 *
 * Build: make -C oracle   ->  oracle/_build/liboracle.so
 */
#define _GNU_SOURCE
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <math.h>
#include <pthread.h>
#include <unistd.h>

/* ------------------------------------------------------------------------------------------------ types */
enum { OT_U8 = 0, OT_I8, OT_U16, OT_I16, OT_U32, OT_I32, OT_U64, OT_I64, OT_F32, OT_F64 };
enum { OP_EQ = 0, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_IN };

typedef struct {
    int32_t col;   /* column index in the storage schema */
    int32_t op;    /* OP_* */
    int64_t i;     /* literal for signed columns */
    uint64_t u;    /* literal for unsigned columns */
    double f;      /* literal for float columns */
    const uint64_t *in_vals;  /* OP_IN: the list, every value in the column's widened domain (i64 / u64 / f64 bits) */
    int32_t in_count, _pad;
} orc_pred;

typedef struct {
    int64_t n;
    int ncols;
    uint64_t **vals; /* widened 8-byte slots: signed ints sign-extended, unsigned zero-extended, floats as f64 bits */
    uint8_t **valid; /* 1 = non-null */
} orc_table;

static __thread char g_err[512];
const char *orc_last_error(void) { return g_err; }
#define FAIL(...) do { snprintf(g_err, sizeof g_err, __VA_ARGS__); return -1; } while (0)

static int type_is_signed(int t) { return t == OT_I8 || t == OT_I16 || t == OT_I32 || t == OT_I64; }
static int type_is_float(int t) { return t == OT_F32 || t == OT_F64; }

static orc_table *table_new(int ncols, int64_t n) {
    orc_table *t = calloc(1, sizeof *t);
    t->n = n; t->ncols = ncols;
    t->vals = calloc(ncols, sizeof *t->vals);
    t->valid = calloc(ncols, sizeof *t->valid);
    for (int c = 0; c < ncols; c++) {
        t->vals[c] = malloc(sizeof(uint64_t) * (n ? n : 1));
        t->valid[c] = malloc(n ? n : 1);
    }
    return t;
}
void orc_table_free(orc_table *t) {
    if (!t) return;
    for (int c = 0; c < t->ncols; c++) { free(t->vals[c]); free(t->valid[c]); }
    free(t->vals); free(t->valid); free(t);
}
int64_t orc_table_rows(const orc_table *t) { return t->n; }
const uint64_t *orc_table_col(const orc_table *t, int c) { return t->vals[c]; }
const uint8_t *orc_table_valid(const orc_table *t, int c) { return t->valid[c]; }

/* ------------------------------------------------------------------------------- Thrift compact protocol */
typedef struct { const uint8_t *p, *end; int err; } tr;

static uint64_t tr_varint(tr *r) {
    uint64_t v = 0; int sh = 0;
    while (r->p < r->end) {
        uint8_t b = *r->p++;
        v |= (uint64_t)(b & 0x7f) << sh;
        if (!(b & 0x80)) return v;
        sh += 7;
        if (sh > 63) break;
    }
    r->err = 1; return 0;
}
static int64_t tr_zigzag(tr *r) { uint64_t v = tr_varint(r); return (int64_t)(v >> 1) ^ -(int64_t)(v & 1); }

/* returns field type (0 = STOP); *fid updated */
static int tr_field(tr *r, int *fid) {
    if (r->p >= r->end) { r->err = 1; return 0; }
    uint8_t b = *r->p++;
    if (b == 0) return 0;
    int delta = b >> 4, type = b & 0x0f;
    if (delta) *fid += delta; else *fid = (int)tr_zigzag(r);
    return type;
}
static void tr_skip(tr *r, int type);
static void tr_skip_struct(tr *r) {
    int fid = 0, t;
    while (!r->err && (t = tr_field(r, &fid))) tr_skip(r, t);
}
static int tr_list(tr *r, int *etype) {
    if (r->p >= r->end) { r->err = 1; return 0; }
    uint8_t b = *r->p++;
    int n = b >> 4; *etype = b & 0x0f;
    if (n == 15) n = (int)tr_varint(r);
    return n;
}
static void tr_skip(tr *r, int type) {
    switch (type) {
    case 1: case 2: break;                       /* bool encoded in the field header */
    case 3: r->p += 1; break;
    case 4: case 5: case 6: (void)tr_varint(r); break;
    case 7: r->p += 8; break;
    case 8: { uint64_t n = tr_varint(r); r->p += n; break; }
    case 9: case 10: {
        int et, n = tr_list(r, &et);
        for (int i = 0; i < n && !r->err; i++) { if (et == 1 || et == 2) r->p += 1; else tr_skip(r, et); }
        break;
    }
    case 11: {
        uint64_t n = tr_varint(r);
        if (n) { uint8_t kv = *r->p++; for (uint64_t i = 0; i < n && !r->err; i++) { tr_skip(r, kv >> 4); tr_skip(r, kv & 15); } }
        break;
    }
    case 12: tr_skip_struct(r); break;
    default: r->err = 1;
    }
    if (r->p > r->end) r->err = 1;
}

/* --------------------------------------------------------------------------------- Parquet metadata model */
typedef struct {
    int phys_type, codec;
    int64_t num_values, data_page_offset, dict_page_offset, total_compressed;
    int has_min, has_max, has_nulls;
    uint8_t minv[8], maxv[8];
    int64_t null_count;
} col_meta;
typedef struct { int64_t num_rows; col_meta *cols; } rg_meta;
typedef struct {
    int ncols;            /* leaf columns */
    int *repetition;      /* per leaf: 0 required, 1 optional */
    int64_t num_rows;
    int nrgs; rg_meta *rgs;
} file_meta;

static void parse_statistics(tr *r, col_meta *cm) {
    int fid = 0, t;
    while (!r->err && (t = tr_field(r, &fid))) {
        if ((fid == 5 || fid == 6) && t == 8) {
            uint64_t n = tr_varint(r);
            if (n <= 8) {
                if (fid == 5) { memset(cm->maxv, 0, 8); memcpy(cm->maxv, r->p, n); cm->has_max = 1; }
                else { memset(cm->minv, 0, 8); memcpy(cm->minv, r->p, n); cm->has_min = 1; }
            }
            r->p += n;
        } else if (fid == 3 && t == 6) { cm->null_count = tr_zigzag(r); cm->has_nulls = 1; }
        else tr_skip(r, t);
    }
}
static void parse_col_meta(tr *r, col_meta *cm) {
    int fid = 0, t;
    cm->dict_page_offset = -1;
    while (!r->err && (t = tr_field(r, &fid))) {
        switch (fid) {
        case 1: cm->phys_type = (int)tr_zigzag(r); break;
        case 4: cm->codec = (int)tr_zigzag(r); break;
        case 5: cm->num_values = tr_zigzag(r); break;
        case 7: cm->total_compressed = tr_zigzag(r); break;
        case 9: cm->data_page_offset = tr_zigzag(r); break;
        case 11: cm->dict_page_offset = tr_zigzag(r); break;
        case 12: parse_statistics(r, cm); break;
        default: tr_skip(r, t);
        }
    }
}
static void parse_col_chunk(tr *r, col_meta *cm) {
    int fid = 0, t;
    while (!r->err && (t = tr_field(r, &fid))) {
        if (fid == 3 && t == 12) parse_col_meta(r, cm); else tr_skip(r, t);
    }
}
static void parse_row_group(tr *r, rg_meta *rg, int ncols) {
    int fid = 0, t;
    rg->cols = calloc(ncols, sizeof(col_meta));
    while (!r->err && (t = tr_field(r, &fid))) {
        if (fid == 1 && t == 9) {
            int et, n = tr_list(r, &et);
            for (int i = 0; i < n && !r->err; i++) {
                if (i < ncols) parse_col_chunk(r, &rg->cols[i]); else tr_skip_struct(r);
            }
        } else if (fid == 3 && t == 6) rg->num_rows = tr_zigzag(r);
        else tr_skip(r, t);
    }
}
static void file_meta_free(file_meta *fm) {
    for (int i = 0; i < fm->nrgs; i++) free(fm->rgs[i].cols);
    free(fm->rgs); free(fm->repetition);
}
static int parse_footer(const uint8_t *data, uint64_t len, file_meta *fm) {
    memset(fm, 0, sizeof *fm);
    if (len < 12 || memcmp(data, "PAR1", 4) || memcmp(data + len - 4, "PAR1", 4)) FAIL("not a parquet file");
    uint32_t mlen; memcpy(&mlen, data + len - 8, 4);
    if ((uint64_t)mlen + 12 > len) FAIL("bad footer length");
    tr r = { data + len - 8 - mlen, data + len - 8, 0 };
    int fid = 0, t;
    while (!r.err && (t = tr_field(&r, &fid))) {
        if (fid == 2 && t == 9) { /* schema: root + leaves (flat schemas only) */
            int et, n = tr_list(&r, &et);
            fm->ncols = n - 1;
            fm->repetition = calloc(n, sizeof(int));
            for (int i = 0; i < n && !r.err; i++) {
                int f2 = 0, t2, rep = 0;
                while (!r.err && (t2 = tr_field(&r, &f2))) {
                    if (f2 == 3 && t2 == 5) rep = (int)tr_zigzag(&r); else tr_skip(&r, t2);
                }
                if (i > 0) fm->repetition[i - 1] = rep;
            }
        } else if (fid == 3 && t == 6) fm->num_rows = tr_zigzag(&r);
        else if (fid == 4 && t == 9) {
            int et, n = tr_list(&r, &et);
            fm->nrgs = n; fm->rgs = calloc(n ? n : 1, sizeof(rg_meta));
            for (int i = 0; i < n && !r.err; i++) parse_row_group(&r, &fm->rgs[i], fm->ncols);
        } else tr_skip(&r, t);
    }
    if (r.err) { file_meta_free(fm); FAIL("thrift parse error in footer"); }
    return 0;
}

typedef struct {
    int type, uncomp, comp;
    int num_values, encoding, def_enc;
    int v2_def_len, v2_rep_len, v2_is_compressed, v2_num_nulls;
    int hdr_len;
} page_hdr;
static int parse_page_header(const uint8_t *p, const uint8_t *end, page_hdr *h) {
    memset(h, 0, sizeof *h); h->v2_is_compressed = 1; h->def_enc = 3;
    tr r = { p, end, 0 };
    int fid = 0, t;
    while (!r.err && (t = tr_field(&r, &fid))) {
        if (fid == 1) h->type = (int)tr_zigzag(&r);
        else if (fid == 2) h->uncomp = (int)tr_zigzag(&r);
        else if (fid == 3) h->comp = (int)tr_zigzag(&r);
        else if ((fid == 5 || fid == 7) && t == 12) {
            int f2 = 0, t2;
            while (!r.err && (t2 = tr_field(&r, &f2))) {
                if (f2 == 1) h->num_values = (int)tr_zigzag(&r);
                else if (f2 == 2) h->encoding = (int)tr_zigzag(&r);
                else if (f2 == 3 && fid == 5) h->def_enc = (int)tr_zigzag(&r);
                else tr_skip(&r, t2);
            }
        } else if (fid == 8 && t == 12) {
            int f2 = 0, t2;
            while (!r.err && (t2 = tr_field(&r, &f2))) {
                if (f2 == 1) h->num_values = (int)tr_zigzag(&r);
                else if (f2 == 2) h->v2_num_nulls = (int)tr_zigzag(&r);
                else if (f2 == 4) h->encoding = (int)tr_zigzag(&r);
                else if (f2 == 5) h->v2_def_len = (int)tr_zigzag(&r);
                else if (f2 == 6) h->v2_rep_len = (int)tr_zigzag(&r);
                else if (f2 == 7) h->v2_is_compressed = (t2 == 1);
                else tr_skip(&r, t2);
            }
        } else tr_skip(&r, t);
    }
    if (r.err) FAIL("thrift parse error in page header");
    h->hdr_len = (int)(r.p - p);
    return 0;
}

/* ----------------------------------------------------------------------------------- Snappy (raw format) */
static int snappy_decompress(const uint8_t *src, int64_t n, uint8_t *dst, int64_t cap) {
    const uint8_t *p = src, *end = src + n;
    uint64_t ulen = 0; int sh = 0;
    while (p < end) { uint8_t b = *p++; ulen |= (uint64_t)(b & 0x7f) << sh; if (!(b & 0x80)) break; sh += 7; }
    if ((int64_t)ulen > cap) FAIL("snappy: output larger than expected");
    int64_t o = 0;
    while (p < end) {
        uint8_t tag = *p++;
        int64_t len; int64_t off;
        switch (tag & 3) {
        case 0:
            len = (tag >> 2) + 1;
            if (len > 60) {
                int nb = (int)len - 60; len = 0;
                if (p + nb > end) FAIL("snappy: truncated literal length");
                for (int i = 0; i < nb; i++) len |= (int64_t)p[i] << (8 * i);
                len += 1; p += nb;
            }
            if (p + len > end || o + len > (int64_t)ulen) FAIL("snappy: literal overrun");
            memcpy(dst + o, p, len); p += len; o += len;
            continue;
        case 1: len = ((tag >> 2) & 7) + 4; off = ((int64_t)(tag >> 5) << 8) | *p++; break;
        case 2: len = (tag >> 2) + 1; off = p[0] | (p[1] << 8); p += 2; break;
        default: len = (tag >> 2) + 1; off = (int64_t)p[0] | ((int64_t)p[1] << 8) | ((int64_t)p[2] << 16) | ((int64_t)p[3] << 24); p += 4;
        }
        if (off == 0 || off > o || o + len > (int64_t)ulen) FAIL("snappy: bad copy");
        for (int64_t i = 0; i < len; i++) dst[o + i] = dst[o + i - off]; /* byte-serial: overlapping copies replicate */
        o += len;
    }
    if (o != (int64_t)ulen) FAIL("snappy: short output");
    return 0;
}

/* -------------------------------------------------------------------------------- Zstandard (RFC 8878) */
#include "zstd_oracle.h"

/* page payload -> uncompressed bytes by Parquet codec id (1 Snappy, 6 Zstandard: ParquetCompression, config.rs:78-94) */
static int page_decompress(int codec, const uint8_t *src, int64_t n, uint8_t *dst, int64_t cap) {
    if (codec == 1) return snappy_decompress(src, n, dst, cap);
    if (codec == 6) return zstd_decompress(src, n, dst, cap);
    FAIL("oracle: unsupported codec %d", codec);
}
/* test hook: one raw codec stream (tests pin the restatement on libsnappy / libzstd streams from pyarrow) */
int orc_decompress(int codec, const uint8_t *src, int64_t n, uint8_t *dst, int64_t cap) { return page_decompress(codec, src, n, dst, cap); }

/* ------------------------------------------------------------------- RLE / bit-packed hybrid (def levels) */
static int decode_levels_bw1(const uint8_t *p, int64_t nbytes, int n, uint8_t *out) {
    const uint8_t *end = p + nbytes;
    int i = 0;
    while (i < n && p < end) {
        uint64_t h = 0; int sh = 0;
        while (p < end) { uint8_t b = *p++; h |= (uint64_t)(b & 0x7f) << sh; if (!(b & 0x80)) break; sh += 7; }
        if (h & 1) { /* bit-packed: (h>>1) groups of 8 one-bit values, LSB first */
            int64_t groups = (int64_t)(h >> 1);
            for (int64_t g = 0; g < groups && p < end; g++) {
                uint8_t b = *p++;
                for (int k = 0; k < 8 && i < n; k++) out[i++] = (b >> k) & 1;
            }
        } else {
            int64_t run = (int64_t)(h >> 1);
            if (p >= end) FAIL("levels: truncated RLE run");
            uint8_t v = *p++ & 1;
            for (int64_t k = 0; k < run && i < n; k++) out[i++] = v;
        }
    }
    if (i != n) FAIL("levels: decoded %d of %d", i, n);
    return 0;
}

/* ---------------------------------------------------------------------------------- page / chunk decoding */
static int phys_width(int phys) { return phys == 1 || phys == 4 ? 4 : (phys == 2 || phys == 5 ? 8 : 0); }

static uint64_t widen(const uint8_t *p, int phys, int otype) {
    if (phys == 1) { /* INT32 */
        int32_t v; memcpy(&v, p, 4);
        switch (otype) {
        case OT_U8: return (uint8_t)v; case OT_U16: return (uint16_t)v; case OT_U32: return (uint32_t)v;
        default: return (uint64_t)(int64_t)v;
        }
    } else if (phys == 2) { uint64_t v; memcpy(&v, p, 8); return v; }
    else if (phys == 4) { float f; memcpy(&f, p, 4); double d = f; uint64_t v; memcpy(&v, &d, 8); return v; }
    else { uint64_t v; memcpy(&v, p, 8); return v; }
}

/* DELTA_BINARY_PACKED (Apache Parquet format spec, Encodings.md; selectable per column through config.rs:54-75):
 * header = block size, miniblocks per block, total count, first value (zigzag); every block = min delta (zigzag), one bit
 * width per miniblock, then the miniblocks' (delta - min delta) bit-packed LSB first.  All sums wrap in the physical width.
 * Decodes `count` values into out[] as PLAIN bytes of width w (4 or 8). */
static int delta_binary_unpack(const uint8_t *p, int64_t len, int w, int64_t count, uint8_t *out) {
    const uint8_t *end = p + len;
#define DVAR(var) do { uint64_t _v = 0; int _s = 0; for (;;) { if (p >= end || _s > 63) FAIL("delta: truncated varint"); uint8_t _b = *p++; _v |= (uint64_t)(_b & 0x7f) << _s; _s += 7; if (!(_b & 0x80)) break; } var = _v; } while (0)
    uint64_t block, nmini, total, zz;
    DVAR(block); DVAR(nmini); DVAR(total); DVAR(zz);
    if (nmini == 0 || block == 0 || block % nmini || (block / nmini) % 32) FAIL("delta: bad block geometry");
    if ((int64_t)total != count) FAIL("delta: %llu values in the page header, %lld expected", (unsigned long long)total, (long long)count);
    uint64_t per = block / nmini;
    uint64_t cur = (zz >> 1) ^ (uint64_t)-(int64_t)(zz & 1);
    int64_t done = 0;
    if (count > 0) { if (w == 4) { uint32_t x = (uint32_t)cur; memcpy(out, &x, 4); } else memcpy(out, &cur, 8); done = 1; }
    while (done < count) {
        uint64_t mz; DVAR(mz);
        uint64_t min_delta = (mz >> 1) ^ (uint64_t)-(int64_t)(mz & 1);
        if (p + nmini > end) FAIL("delta: truncated bit widths");
        const uint8_t *bw = p; p += nmini;
        for (uint64_t m = 0; m < nmini && done < count; m++) {
            int b = bw[m];
            if (b > 64) FAIL("delta: bit width %d", b);
            if (p + per * b / 8 > end) FAIL("delta: truncated miniblock");
            for (uint64_t j = 0; j < per && done < count; j++) {
                uint64_t bit = j * (uint64_t)b, v = 0;
                for (int k = 0; k < b; k++) { uint64_t q = bit + k; v |= (uint64_t)((p[q >> 3] >> (q & 7)) & 1) << k; }
                cur += min_delta + v;
                if (w == 4) { uint32_t x = (uint32_t)cur; memcpy(out + done * 4, &x, 4); cur = (uint64_t)(int64_t)(int32_t)x; }
                else memcpy(out + done * 8, &cur, 8);
                done++;
            }
            p += per * b / 8;
        }
    }
#undef DVAR
    return 0;
}

/* RLE_DICTIONARY / PLAIN_DICTIONARY data page (enable_dict, config.rs:98-103,127): [bit width : 1 byte] then RLE / bit-packed
 * hybrid runs of dictionary indices (Parquet Encodings.md); out[i] = dict[index_i] as PLAIN bytes of width w. */
static int dict_indices_unpack(const uint8_t *p, int64_t len, int w, int64_t count, const uint8_t *dict, int64_t dict_n, uint8_t *out) {
    const uint8_t *end = p + len;
    if (count == 0) return 0;
    if (p >= end) FAIL("dict: empty data page");
    int bw = *p++;
    if (bw > 32) FAIL("dict: bit width %d", bw);
    int64_t i = 0;
    while (i < count) {
        uint64_t h = 0; int sh = 0;
        for (;;) { if (p >= end) FAIL("dict: truncated run header"); uint8_t b = *p++; h |= (uint64_t)(b & 0x7f) << sh; if (!(b & 0x80)) break; sh += 7; }
        if (h & 1) {                               /* bit-packed: groups of 8 indices */
            int64_t groups = (int64_t)(h >> 1);
            if (p + groups * bw > end) FAIL("dict: truncated bit-packed run");
            for (int64_t k = 0; k < groups * 8 && i < count; k++, i++) {
                uint64_t bit = (uint64_t)k * bw, idx = 0;
                for (int b = 0; b < bw; b++) { uint64_t q = bit + b; idx |= (uint64_t)((p[q >> 3] >> (q & 7)) & 1) << b; }
                if ((int64_t)idx >= dict_n) FAIL("dict: index out of range");
                memcpy(out + i * w, dict + idx * w, w);
            }
            p += groups * bw;
        } else {
            int64_t run = (int64_t)(h >> 1);
            int nb = (bw + 7) / 8;
            if (p + nb > end) FAIL("dict: truncated RLE run");
            uint64_t idx = 0;
            for (int b = 0; b < nb; b++) idx |= (uint64_t)p[b] << (8 * b);
            p += nb;
            if (run > 0 && (int64_t)idx >= dict_n) FAIL("dict: index out of range");
            for (int64_t k = 0; k < run && i < count; k++, i++) memcpy(out + i * w, dict + idx * w, w);
            if (run == 0) FAIL("dict: empty run");
        }
    }
    return 0;
}

/* decode one column chunk into vals/valid[0..num_rows) */
static int decode_chunk(const uint8_t *data, uint64_t len, const col_meta *cm, int optional, int otype,
                        int64_t num_rows, uint64_t *vals, uint8_t *valid) {
    int w = phys_width(cm->phys_type);
    if (!w) FAIL("oracle: unsupported physical type %d", cm->phys_type);
    if (cm->codec != 0 && cm->codec != 1 && cm->codec != 6) FAIL("oracle: unsupported codec %d", cm->codec);
    int64_t pos = cm->data_page_offset, row = 0;
    if (cm->dict_page_offset > 0 && cm->dict_page_offset < cm->data_page_offset) pos = cm->dict_page_offset;   /* dictionary page first */
    uint8_t *buf = NULL; int64_t bufcap = 0;
    uint8_t *dict = NULL; int64_t dict_n = 0;
    uint8_t *lv = malloc(num_rows ? num_rows : 1);
    int rc = 0;
    while (row < num_rows) {
        page_hdr h;
        if ((uint64_t)pos >= len) { rc = -1; snprintf(g_err, sizeof g_err, "page offset out of file"); break; }
        if (parse_page_header(data + pos, data + len, &h)) { rc = -1; break; }
        const uint8_t *payload = data + pos + h.hdr_len;
        pos += h.hdr_len + h.comp;
        if (h.type == 2) {                        /* dictionary page: PLAIN values, compressed like a data page */
            free(dict);
            dict = malloc((size_t)(h.uncomp > 0 ? h.uncomp : 1));
            if (cm->codec != 0) { if (page_decompress(cm->codec, payload, h.comp, dict, h.uncomp)) { rc = -1; break; } }
            else memcpy(dict, payload, (size_t)h.comp);
            dict_n = h.uncomp / w;
            continue;
        }
        if (h.type != 0 && h.type != 3) continue;
        if (h.encoding != 0 && !(h.encoding == 5 && (cm->phys_type == 1 || cm->phys_type == 2)) && !((h.encoding == 8 || h.encoding == 2) && dict)) {
            rc = -1; snprintf(g_err, sizeof g_err, "oracle: encoding %d unsupported", h.encoding); break;
        }
        if (h.type == 0 && optional && h.def_enc != 3) {  /* deprecated BIT_PACKED levels: no length in front, not read */
            rc = -1; snprintf(g_err, sizeof g_err, "oracle: definition level encoding %d unsupported", h.def_enc); break;
        }
        int nv = h.num_values;
        if (row + nv > num_rows) { rc = -1; snprintf(g_err, sizeof g_err, "page rows overflow chunk"); break; }
        const uint8_t *body; int64_t body_len;
        const uint8_t *levels = NULL; int64_t levels_len = 0;
        if (h.type == 0) { /* V1: whole payload compressed */
            if (cm->codec != 0) {
                if (h.uncomp > bufcap) { bufcap = h.uncomp + 64; buf = realloc(buf, bufcap); }
                if (page_decompress(cm->codec, payload, h.comp, buf, h.uncomp)) { rc = -1; break; }
                body = buf; body_len = h.uncomp;
            } else { body = payload; body_len = h.comp; }
            if (optional) {
                uint32_t ll; memcpy(&ll, body, 4);
                levels = body + 4; levels_len = ll; body += 4 + ll; body_len -= 4 + ll;
            }
        } else { /* V2: levels stored uncompressed ahead of the (optionally compressed) values */
            levels = payload + h.v2_rep_len; levels_len = h.v2_def_len;
            const uint8_t *vsrc = payload + h.v2_rep_len + h.v2_def_len;
            int64_t vcomp = h.comp - h.v2_rep_len - h.v2_def_len, vun = h.uncomp - h.v2_rep_len - h.v2_def_len;
            if (cm->codec != 0 && h.v2_is_compressed) {
                if (vun > bufcap) { bufcap = vun + 64; buf = realloc(buf, bufcap); }
                if (page_decompress(cm->codec, vsrc, vcomp, buf, vun)) { rc = -1; break; }
                body = buf; body_len = vun;
            } else { body = vsrc; body_len = vcomp; }
        }
        if (optional) { if (decode_levels_bw1(levels, levels_len, nv, lv)) { rc = -1; break; } }
        else memset(lv, 1, nv);
        uint8_t *dbuf = NULL;
        if (h.encoding == 5) {                    /* DELTA_BINARY_PACKED: expand to PLAIN bytes, then the common path */
            int64_t nn = 0;
            for (int i = 0; i < nv; i++) nn += lv[i] != 0;
            dbuf = malloc((size_t)(nn ? nn : 1) * w);
            if (delta_binary_unpack(body, body_len, w, nn, dbuf)) { free(dbuf); rc = -1; break; }
            body = dbuf; body_len = nn * w;
        }
        if (h.encoding == 8 || h.encoding == 2) { /* dictionary indices: expand to PLAIN bytes, then the common path */
            int64_t nn = 0;
            for (int i = 0; i < nv; i++) nn += lv[i] != 0;
            dbuf = malloc((size_t)(nn ? nn : 1) * w);
            if (dict_indices_unpack(body, body_len, w, nn, dict, dict_n, dbuf)) { free(dbuf); rc = -1; break; }
            body = dbuf; body_len = nn * w;
        }
        int64_t k = 0;
        for (int i = 0; i < nv; i++) {
            if (lv[i]) {
                if ((k + 1) * w > body_len) { rc = -1; snprintf(g_err, sizeof g_err, "PLAIN values truncated"); break; }
                vals[row + i] = widen(body + k * w, cm->phys_type, otype); valid[row + i] = 1; k++;
            } else { vals[row + i] = 0; valid[row + i] = 0; }
        }
        free(dbuf);
        if (rc) break;
        row += nv;
    }
    free(buf); free(lv); free(dict);
    return rc;
}

/* ---------------------------------------------------------------------------------------- typed compares */
static int cmp_typed(uint64_t a, uint64_t b, int t) {
    /* arrow-rs 53 comparison kernels (behind FilterExec / PruningPredicate, read.rs:459-470) order floats by IEEE-754
       totalOrder: NaN is above +inf (below -inf when its sign bit is set) and -0.0 < +0.0 */
    if (type_is_float(t)) {
        uint64_t x = a ^ ((a >> 63) ? ~(uint64_t)0 : ((uint64_t)1 << 63)), y = b ^ ((b >> 63) ? ~(uint64_t)0 : ((uint64_t)1 << 63));
        return x < y ? -1 : (x > y ? 1 : 0);
    }
    if (type_is_signed(t)) { int64_t x = (int64_t)a, y = (int64_t)b; return x < y ? -1 : (x > y ? 1 : 0); }
    return a < b ? -1 : (a > b ? 1 : 0);
}
static uint64_t pred_literal(const orc_pred *p, int t) {
    if (type_is_float(t)) { uint64_t v; memcpy(&v, &p->f, 8); return v; }
    if (type_is_signed(t)) return (uint64_t)p->i;
    return p->u;
}
static int pred_eval(const orc_pred *p, int t, uint64_t v) {
    if (p->op == OP_IN) {                       /* `col IN (v1, ..)`: DataFusion's InListExpr, NULL handled by the caller (NULL => false) */
        for (int i = 0; i < p->in_count; i++) if (cmp_typed(v, p->in_vals[i], t) == 0) return 1;
        return 0;
    }
    int c = cmp_typed(v, pred_literal(p, t), t);
    switch (p->op) {
    case OP_EQ: return c == 0; case OP_NE: return c != 0; case OP_LT: return c < 0;
    case OP_LE: return c <= 0; case OP_GT: return c > 0; default: return c >= 0;
    }
}
/* DataFusion PruningPredicate rewrite (read.rs:613 pins the Eq form): may this row group contain matches? */
static uint64_t stat_widen(const uint8_t *raw, int phys, int t) { return widen(raw, phys, t); }
static int rg_may_match(const rg_meta *rg, const orc_pred *preds, int np, const int *types) {
    for (int i = 0; i < np; i++) {
        const col_meta *cm = &rg->cols[preds[i].col];
        int t = types[preds[i].col];
        if (cm->has_nulls && cm->null_count == rg->num_rows) return 0; /* CASE WHEN null_count = row_count THEN false */
        if (!cm->has_min || !cm->has_max) continue;
        uint64_t mn = stat_widen(cm->minv, cm->phys_type, t), mx = stat_widen(cm->maxv, cm->phys_type, t);
        uint64_t lit = pred_literal(&preds[i], t);
        int ok = 1;
        switch (preds[i].op) {
        case OP_EQ: ok = cmp_typed(mn, lit, t) <= 0 && cmp_typed(lit, mx, t) <= 0; break;
        case OP_NE: ok = cmp_typed(mn, lit, t) != 0 || cmp_typed(lit, mx, t) != 0; break;
        case OP_LT: ok = cmp_typed(mn, lit, t) < 0; break;
        case OP_LE: ok = cmp_typed(mn, lit, t) <= 0; break;
        case OP_GT: ok = cmp_typed(mx, lit, t) > 0; break;
        case OP_GE: ok = cmp_typed(mx, lit, t) >= 0; break;
        case OP_IN:   /* PruningPredicate rewrites a short IN list into `c = v1 OR c = v2 ..`: some value inside [min, max] */
            ok = 0;
            for (int j = 0; j < preds[i].in_count && !ok; j++)
                ok = cmp_typed(mn, preds[i].in_vals[j], t) <= 0 && cmp_typed(preds[i].in_vals[j], mx, t) <= 0;
            break;
        }
        if (!ok) return 0;
    }
    return 1;
}

/* ------------------------------------------------------------------- S2+S3: one SST -> filtered row stream */
typedef struct {
    orc_table *t;           /* filtered rows */
    int64_t *chunk_end;     /* passthrough batch boundaries (k == 1): end offset of each non-empty reader batch */
    int nchunks;
    int64_t rows_in_file, rows_decoded;
} sst_stream;

static int decode_filter_sst(const uint8_t *data, uint64_t len, int ncols, const int *types,
                             const orc_pred *preds, int np, int prune, int batch_size, sst_stream *out) {
    file_meta fm;
    memset(out, 0, sizeof *out);
    if (parse_footer(data, len, &fm)) return -1;
    if (fm.ncols != ncols) { file_meta_free(&fm); FAIL("schema mismatch: file has %d columns, expected %d", fm.ncols, ncols); }
    int64_t total = 0;
    for (int g = 0; g < fm.nrgs; g++) total += fm.rgs[g].num_rows;
    out->rows_in_file = total;
    orc_table *t = table_new(ncols, total);
    out->chunk_end = malloc(sizeof(int64_t) * (total / (batch_size > 0 ? batch_size : 1) + fm.nrgs + 2));
    int64_t w = 0;
    uint64_t **tv = malloc(sizeof(*tv) * ncols); uint8_t **tb = malloc(sizeof(*tb) * ncols);
    int rc = 0;
    for (int g = 0; g < fm.nrgs && !rc; g++) {
        rg_meta *rg = &fm.rgs[g];
        if (prune && np && !rg_may_match(rg, preds, np, types)) continue;
        int64_t n = rg->num_rows;
        out->rows_decoded += n;
        for (int c = 0; c < ncols; c++) { tv[c] = malloc(8 * (n ? n : 1)); tb[c] = malloc(n ? n : 1); }
        for (int c = 0; c < ncols && !rc; c++)
            rc = decode_chunk(data, len, &rg->cols[c], fm.repetition[c] == 1, types[c], n, tv[c], tb[c]);
        /* parquet reader yields <= batch_size rows per batch inside a row group; FilterExec filters each batch */
        for (int64_t b0 = 0; b0 < n && !rc; b0 += batch_size) {
            int64_t b1 = b0 + batch_size < n ? b0 + batch_size : n, w0 = w;
            for (int64_t r = b0; r < b1; r++) {
                int keep = 1;
                for (int i = 0; i < np && keep; i++) {
                    int c = preds[i].col;
                    keep = tb[c][r] && pred_eval(&preds[i], types[c], tv[c][r]); /* NULL => false */
                }
                if (keep) { for (int c = 0; c < ncols; c++) { t->vals[c][w] = tv[c][r]; t->valid[c][w] = tb[c][r]; } w++; }
            }
            if (w > w0) out->chunk_end[out->nchunks++] = w;
        }
        for (int c = 0; c < ncols; c++) { free(tv[c]); free(tb[c]); }
    }
    free(tv); free(tb);
    t->n = w; out->t = t;
    file_meta_free(&fm);
    if (rc) { orc_table_free(t); free(out->chunk_end); out->t = NULL; out->chunk_end = NULL; }
    return rc;
}

int orc_decode_sst(const uint8_t *data, uint64_t len, int ncols, const int *types,
                   const orc_pred *preds, int np, int prune, orc_table **out) {
    sst_stream s;
    if (decode_filter_sst(data, len, ncols, types, preds, np, prune, 8192, &s)) return -1;
    free(s.chunk_end); *out = s.t; return 0;
}

/* ---------------------------------------------------------------- S4: k-way merge on (pk..., __seq__) */
typedef struct { int src; int64_t row; } rowref;
typedef struct { sst_stream *s; int k, num_pk, seq_idx; const int *types; } merge_ctx;

/* ASC NULLS FIRST per column (read.rs:412-427); ties -> lower stream index */
static int row_less(const merge_ctx *m, int sa, int64_t ra, int sb, int64_t rb) {
    const orc_table *a = m->s[sa].t, *b = m->s[sb].t;
    for (int c = 0; c <= m->num_pk; c++) {
        int col = c < m->num_pk ? c : m->seq_idx;
        int va = a->valid[col][ra], vb = b->valid[col][rb];
        if (va != vb) return va < vb;            /* null first */
        if (!va) continue;
        int d = cmp_typed(a->vals[col][ra], b->vals[col][rb], m->types[col]);
        if (d) return d < 0;
    }
    return sa < sb;
}

static rowref *kway_merge(merge_ctx *m, int64_t *n_out) {
    int64_t total = 0;
    for (int i = 0; i < m->k; i++) total += m->s[i].t->n;
    rowref *out = malloc(sizeof(rowref) * (total ? total : 1));
    int *heap = malloc(sizeof(int) * (m->k + 1)); int64_t *cur = calloc(m->k, sizeof(int64_t)); int hn = 0;
#define HLESS(x, y) row_less(m, x, cur[x], y, cur[y])
    for (int i = 0; i < m->k; i++) if (m->s[i].t->n > 0) {
        int j = hn++; heap[j] = i;
        while (j > 0) { int p = (j - 1) / 2; if (HLESS(heap[j], heap[p])) { int t = heap[j]; heap[j] = heap[p]; heap[p] = t; j = p; } else break; }
    }
    int64_t w = 0;
    while (hn > 0) {
        int s = heap[0];
        out[w].src = s; out[w].row = cur[s]; w++;
        if (++cur[s] >= m->s[s].t->n) heap[0] = heap[--hn];
        int j = 0;
        for (;;) {
            int l = 2 * j + 1, r = l + 1, b = j;
            if (l < hn && HLESS(heap[l], heap[b])) b = l;
            if (r < hn && HLESS(heap[r], heap[b])) b = r;
            if (b == j) break;
            int t = heap[j]; heap[j] = heap[b]; heap[b] = t; j = b;
        }
    }
#undef HLESS
    free(heap); free(cur);
    *n_out = w; return out;
}

/* ------------------------------------------------------- S5/S6: MergeStream over the merged, chunked stream */
/* primary_key_eq (read.rs:262-287): value-only comparison (null bitmap ignored); PK types outside
 * {U8,I8,U32,I32,U64,I64} fall through to `true` in the reference (SURVEY §8 S5) — reproduced. */
static int pk_eq(const merge_ctx *m, rowref a, rowref b) {
    for (int c = 0; c < m->num_pk; c++) {
        int t = m->types[c];
        if (t == OT_U16 || t == OT_I16 || t == OT_F32 || t == OT_F64) continue;
        if (m->s[a.src].t->vals[c][a.row] != m->s[b.src].t->vals[c][b.row]) return 0;
    }
    return 1;
}

/* Returns surviving row refs (LastValue) and the output batch boundaries. */
static rowref *merge_stream(const merge_ctx *m, const rowref *in, int64_t n, const int64_t *chunk_end, int nchunks,
                            int64_t *n_out, int64_t **batch_end_out, int *nbatches_out) {
    rowref *out = malloc(sizeof(rowref) * (n ? n : 1));
    int64_t *bend = malloc(sizeof(int64_t) * (nchunks + 2));
    int nb = 0; int64_t w = 0;
    int have_pending = 0; int64_t pend_lo = 0, pend_hi = 0; /* pending_batch = merged rows [pend_lo, pend_hi) */
    int64_t c0 = 0;
    for (int ci = 0; ci < nchunks; ci++) {
        int64_t c1 = chunk_end[ci];
        if (c1 == c0) continue;                       /* merge_batch: empty batch -> None (read.rs:290-292) */
        int64_t w0 = w;
        /* group rows with the same primary keys (read.rs:295-306) */
        int64_t first_run_end = c0 + 1;
        while (first_run_end < c1 && pk_eq(m, in[c0], in[first_run_end])) first_run_end++;
        int64_t last_run_start = c0; /* start of the tail run */
        { int64_t s = c0; while (s < c1) { int64_t e = s + 1; while (e < c1 && pk_eq(m, in[s], in[e])) e++; last_run_start = s; s = e; } }
        int64_t head_lo = c0; /* logical start of the head run after joining with pending */
        if (have_pending) {
            if (pk_eq(m, in[pend_hi - 1], in[c0])) head_lo = pend_lo;           /* concat(pending, head run) */
            else out[w++] = in[pend_hi - 1];                                    /* operator.merge(pending) */
            have_pending = 0;
        }
        /* tail run is held back as pending_batch (read.rs:327-329) */
        if (last_run_start == c0) { pend_lo = head_lo; pend_hi = c1; }          /* single run: popped run is the joined head */
        else { pend_lo = last_run_start; pend_hi = c1; }
        have_pending = 1;
        /* every remaining run -> LastValue = its last row (operator.rs:39-44) */
        { int64_t s = c0; while (s < last_run_start) { int64_t e = s + 1; while (e < c1 && pk_eq(m, in[s], in[e])) e++; out[w++] = in[e - 1]; s = e; } }
        if (w > w0) bend[nb++] = w;                   /* output_batches.is_empty() -> None (read.rs:334-336) */
        c0 = c1;
        (void)first_run_end;
    }
    if (have_pending) { out[w++] = in[pend_hi - 1]; bend[nb++] = w; }           /* poll_next final flush (read.rs:356-367) */
    *n_out = w; *batch_end_out = bend; *nbatches_out = nb;
    return out;
}

/* ------------------------------------------------------------------------------------------ public: scan */
typedef struct {
    orc_table *rows;         /* output rows (builtin columns stripped unless keep_builtin) */
    int64_t *batch_end; int nbatches;
    int64_t rows_in_files, rows_decoded, rows_filtered, rows_merged;
} orc_scan_result;

void orc_scan_result_free(orc_scan_result *r) { if (!r) return; orc_table_free(r->rows); free(r->batch_end); free(r); }
orc_table *orc_scan_rows(orc_scan_result *r) { return r->rows; }
int orc_scan_nbatches(orc_scan_result *r) { return r->nbatches; }
const int64_t *orc_scan_batch_end(orc_scan_result *r) { return r->batch_end; }
int64_t orc_scan_stat(orc_scan_result *r, int which) {
    switch (which) { case 0: return r->rows_in_files; case 1: return r->rows_decoded; case 2: return r->rows_filtered; default: return r->rows_merged; }
}

typedef struct {
    const uint8_t **datas; const uint64_t *lens; int k, ncols; const int *types; const orc_pred *preds; int np, prune, batch_size;
    sst_stream *st; int next; int rc; char *errbuf; pthread_mutex_t mu;
} decode_job;
static void *decode_worker(void *arg) {
    decode_job *j = arg;
    for (;;) {
        pthread_mutex_lock(&j->mu); int i = j->next++; pthread_mutex_unlock(&j->mu);
        if (i >= j->k) break;
        if (decode_filter_sst(j->datas[i], j->lens[i], j->ncols, j->types, j->preds, j->np, j->prune, j->batch_size, &j->st[i])) {
            pthread_mutex_lock(&j->mu); j->rc = -1; snprintf(j->errbuf, 512, "%s", g_err); pthread_mutex_unlock(&j->mu);
        }
    }
    return NULL;
}

static int scan_core(const uint8_t **datas, const uint64_t *lens, int k, int ncols, const int *types, int num_pk,
                     const orc_pred *preds, int np, int batch_size, int prune, int threads,
                     sst_stream **streams_out, rowref **surv_out, int64_t *nsurv_out,
                     int64_t **bend_out, int *nb_out, int64_t stats[4]) {
    sst_stream *st = calloc(k ? k : 1, sizeof *st);
    int rc = 0;
    if (threads < 1) threads = 1;
    /* one partition per SST decodes in parallel (read.rs:442-450); merge + dedup is single-threaded (read.rs:154-156) */
    char errbuf[512] = "";
    decode_job job = { datas, lens, k, ncols, types, preds, np, prune, batch_size, st, 0, 0, errbuf };
    pthread_mutex_init(&job.mu, NULL);
    if (threads > k) threads = k;
    if (threads <= 1) decode_worker(&job);
    else {
        pthread_t *th = malloc(sizeof(pthread_t) * threads);
        for (int i = 0; i < threads; i++) pthread_create(&th[i], NULL, decode_worker, &job);
        for (int i = 0; i < threads; i++) pthread_join(th[i], NULL);
        free(th);
    }
    pthread_mutex_destroy(&job.mu);
    rc = job.rc;
    if (rc) { snprintf(g_err, sizeof g_err, "%s", errbuf); for (int i = 0; i < k; i++) { orc_table_free(st[i].t); free(st[i].chunk_end); } free(st); return -1; }
    memset(stats, 0, 4 * sizeof(int64_t));
    for (int i = 0; i < k; i++) { stats[0] += st[i].rows_in_file; stats[1] += st[i].rows_decoded; stats[2] += st[i].t->n; }
    merge_ctx m = { st, k, num_pk, ncols - 2, types };
    int64_t nm = 0; rowref *merged; int64_t *chunk_end; int nchunks;
    if (k == 1) { /* SortPreservingMergeExec with one input partition is a pass-through: reader batches survive */
        nm = st[0].t->n; merged = malloc(sizeof(rowref) * (nm ? nm : 1));
        for (int64_t r = 0; r < nm; r++) { merged[r].src = 0; merged[r].row = r; }
        nchunks = st[0].nchunks; chunk_end = malloc(sizeof(int64_t) * (nchunks + 1));
        memcpy(chunk_end, st[0].chunk_end, sizeof(int64_t) * nchunks);
    } else {
        merged = kway_merge(&m, &nm);
        nchunks = (int)((nm + batch_size - 1) / batch_size); chunk_end = malloc(sizeof(int64_t) * (nchunks + 1));
        for (int c = 0; c < nchunks; c++) { int64_t e = (int64_t)(c + 1) * batch_size; chunk_end[c] = e < nm ? e : nm; }
    }
    stats[3] = nm;
    *surv_out = merge_stream(&m, merged, nm, chunk_end, nchunks, nsurv_out, bend_out, nb_out);
    free(merged); free(chunk_end);
    *streams_out = st;
    return 0;
}

int orc_scan(const uint8_t **datas, const uint64_t *lens, int k, int ncols, const int *types, int num_pk,
             const orc_pred *preds, int np, int keep_builtin, int batch_size, int prune, int threads,
             orc_scan_result **out) {
    sst_stream *st; rowref *surv; int64_t ns; int64_t *bend; int nb; int64_t stats[4];
    if (batch_size <= 0) batch_size = 8192;
    if (scan_core(datas, lens, k, ncols, types, num_pk, preds, np, batch_size, prune, threads, &st, &surv, &ns, &bend, &nb, stats)) return -1;
    int oc = keep_builtin ? ncols : ncols - 2;        /* maybe_remove_builtin_columns (read.rs:251-260) */
    orc_table *t = table_new(oc, ns);
    for (int c = 0; c < oc; c++)
        for (int64_t r = 0; r < ns; r++) {
            t->vals[c][r] = st[surv[r].src].t->vals[c][surv[r].row];
            t->valid[c][r] = st[surv[r].src].t->valid[c][surv[r].row];
        }
    orc_scan_result *res = calloc(1, sizeof *res);
    res->rows = t; res->batch_end = bend; res->nbatches = nb;
    res->rows_in_files = stats[0]; res->rows_decoded = stats[1]; res->rows_filtered = stats[2]; res->rows_merged = stats[3];
    for (int i = 0; i < k; i++) { orc_table_free(st[i].t); free(st[i].chunk_end); }
    free(st); free(surv);
    *out = res; return 0;
}

/* --------------------------------------------------------------------------------- public: scan+aggregate */
typedef struct {
    int64_t ngroups;
    uint64_t *gkey;     /* group column value (widened) */
    int64_t *bucket;    /* bucket start = ts / w * w (truncate_by, types.rs:82-85); 0 when not windowed */
    uint64_t *count;    /* count(*) over post-dedup rows */
    double *sum, *min, *max;
    int64_t rows_in_files, rows_decoded, rows_filtered, rows_merged, rows_out;
} orc_agg_result;

void orc_agg_result_free(orc_agg_result *a) {
    if (!a) return; free(a->gkey); free(a->bucket); free(a->count); free(a->sum); free(a->min); free(a->max); free(a);
}
int64_t orc_agg_ngroups(orc_agg_result *a) { return a->ngroups; }
const uint64_t *orc_agg_gkey(orc_agg_result *a) { return a->gkey; }
const int64_t *orc_agg_bucket(orc_agg_result *a) { return a->bucket; }
const uint64_t *orc_agg_count(orc_agg_result *a) { return a->count; }
const double *orc_agg_sum(orc_agg_result *a) { return a->sum; }
const double *orc_agg_min(orc_agg_result *a) { return a->min; }
const double *orc_agg_max(orc_agg_result *a) { return a->max; }
int64_t orc_agg_stat(orc_agg_result *a, int which) {
    switch (which) { case 0: return a->rows_in_files; case 1: return a->rows_decoded; case 2: return a->rows_filtered; case 3: return a->rows_merged; default: return a->rows_out; }
}

static double slot_to_double(uint64_t v, int t) {
    if (type_is_float(t)) { double d; memcpy(&d, &v, 8); return d; }
    if (type_is_signed(t)) return (double)(int64_t)v;
    return (double)v;
}

/* group_col < 0: one global group.  ts_col < 0 or window_ms <= 0: no time bucketing.  value_col < 0: count only.
 * Groups are maximal runs of equal (group value, bucket) in the post-dedup stream (sorted by (pk..), so for
 * group_col = pk0 and ts_col = pk1 this is GROUP BY series_id, bucket in key order). */
int orc_scan_aggregate(const uint8_t **datas, const uint64_t *lens, int k, int ncols, const int *types, int num_pk,
                       const orc_pred *preds, int np, int prune, int threads,
                       int group_col, int ts_col, int64_t window_ms, int value_col,
                       orc_agg_result **out) {
    sst_stream *st; rowref *surv; int64_t ns; int64_t *bend; int nb; int64_t stats[4];
    if (scan_core(datas, lens, k, ncols, types, num_pk, preds, np, 8192, prune, threads, &st, &surv, &ns, &bend, &nb, stats)) return -1;
    free(bend);
    orc_agg_result *a = calloc(1, sizeof *a);
    int64_t cap = ns ? ns : 1;
    a->gkey = malloc(8 * cap); a->bucket = malloc(8 * cap); a->count = malloc(8 * cap);
    a->sum = malloc(8 * cap); a->min = malloc(8 * cap); a->max = malloc(8 * cap);
    int64_t g = -1; uint64_t cur_k = 0; int64_t cur_b = 0; int seen_value = 0;
    for (int64_t r = 0; r < ns; r++) {
        const orc_table *t = st[surv[r].src].t; int64_t row = surv[r].row;
        uint64_t kv = group_col >= 0 ? t->vals[group_col][row] : 0;
        int64_t b = 0;
        if (ts_col >= 0 && window_ms > 0) { int64_t ts = (int64_t)t->vals[ts_col][row]; b = ts / window_ms * window_ms; }
        if (g < 0 || kv != cur_k || b != cur_b) {
            g++; cur_k = kv; cur_b = b; seen_value = 0;
            a->gkey[g] = kv; a->bucket[g] = b; a->count[g] = 0; a->sum[g] = 0.0; a->min[g] = INFINITY; a->max[g] = -INFINITY;
        }
        a->count[g]++;
        if (value_col >= 0 && t->valid[value_col][row]) {
            double v = slot_to_double(t->vals[value_col][row], types[value_col]);
            a->sum[g] += v;                                 /* sequential addition in stream order, accumulator starts at 0.0 */
            if (!seen_value || v < a->min[g]) a->min[g] = v;
            if (!seen_value || v > a->max[g]) a->max[g] = v;
            seen_value = 1;
        }
    }
    a->ngroups = g + 1;
    a->rows_in_files = stats[0]; a->rows_decoded = stats[1]; a->rows_filtered = stats[2]; a->rows_merged = stats[3]; a->rows_out = ns;
    for (int i = 0; i < k; i++) { orc_table_free(st[i].t); free(st[i].chunk_end); }
    free(st); free(surv);
    *out = a; return 0;
}

/* GROUP BY for keys that are not a prefix of the sort order (mode "hash"): every surviving row updates the accumulator
 * of its (group value, bucket) in STREAM order — what a single-partition hash aggregation over the reference's scan output
 * computes (the stage is todo!() in the reference, metric_engine/src/metric/mod.rs:37-49) — and the groups are emitted
 * sorted by (group value in its type's order, bucket). */
typedef struct { uint64_t k; int64_t b; int64_t gid; } hslot;
static uint64_t hmix(uint64_t k, int64_t b) {
    uint64_t z = k * 0x9E3779B97F4A7C15ull ^ ((uint64_t)b + 0x632BE59BD9B4E019ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31);
}
static int g_sort_type;
static const orc_agg_result *g_sort_res;
static int cmp_group_ids(const void *x, const void *y) {
    int64_t a = *(const int64_t *)x, b = *(const int64_t *)y;
    int c = cmp_typed(g_sort_res->gkey[a], g_sort_res->gkey[b], g_sort_type);
    if (c) return c;
    return g_sort_res->bucket[a] < g_sort_res->bucket[b] ? -1 : (g_sort_res->bucket[a] > g_sort_res->bucket[b] ? 1 : 0);
}
int orc_scan_aggregate_hash(const uint8_t **datas, const uint64_t *lens, int k, int ncols, const int *types, int num_pk,
                            const orc_pred *preds, int np, int prune, int threads,
                            int group_col, int ts_col, int64_t window_ms, int value_col,
                            orc_agg_result **out) {
    sst_stream *st; rowref *surv; int64_t ns; int64_t *bend; int nb; int64_t stats[4];
    if (scan_core(datas, lens, k, ncols, types, num_pk, preds, np, 8192, prune, threads, &st, &surv, &ns, &bend, &nb, stats)) return -1;
    free(bend);
    orc_agg_result *a = calloc(1, sizeof *a);
    int64_t cap = 1024, ng = 0;
    a->gkey = malloc(8 * cap); a->bucket = malloc(8 * cap); a->count = malloc(8 * cap);
    a->sum = malloc(8 * cap); a->min = malloc(8 * cap); a->max = malloc(8 * cap);
    uint8_t *seen = malloc(cap);
    int64_t hcap = 4096;
    hslot *ht = malloc(sizeof(hslot) * hcap);
    for (int64_t i = 0; i < hcap; i++) ht[i].gid = -1;
    int64_t cur_g = -1; uint64_t cur_k = 0; int64_t cur_b = 0;
    for (int64_t r = 0; r < ns; r++) {
        const orc_table *t = st[surv[r].src].t; int64_t row = surv[r].row;
        uint64_t kv = group_col >= 0 ? t->vals[group_col][row] : 0;
        int64_t b = 0;
        if (ts_col >= 0 && window_ms > 0) { int64_t ts = (int64_t)t->vals[ts_col][row]; b = ts / window_ms * window_ms; }
        if (cur_g < 0 || kv != cur_k || b != cur_b) {
            if ((ng + 1) * 2 > hcap) {                       /* grow + rehash */
                int64_t nc = hcap * 2; hslot *nt = malloc(sizeof(hslot) * nc);
                for (int64_t i = 0; i < nc; i++) nt[i].gid = -1;
                for (int64_t i = 0; i < hcap; i++) if (ht[i].gid >= 0) {
                    uint64_t h = hmix(ht[i].k, ht[i].b) & (uint64_t)(nc - 1);
                    while (nt[h].gid >= 0) h = (h + 1) & (uint64_t)(nc - 1);
                    nt[h] = ht[i];
                }
                free(ht); ht = nt; hcap = nc;
            }
            uint64_t h = hmix(kv, b) & (uint64_t)(hcap - 1);
            while (ht[h].gid >= 0 && !(ht[h].k == kv && ht[h].b == b)) h = (h + 1) & (uint64_t)(hcap - 1);
            if (ht[h].gid < 0) {
                if (ng == cap) {
                    cap *= 2;
                    a->gkey = realloc(a->gkey, 8 * cap); a->bucket = realloc(a->bucket, 8 * cap); a->count = realloc(a->count, 8 * cap);
                    a->sum = realloc(a->sum, 8 * cap); a->min = realloc(a->min, 8 * cap); a->max = realloc(a->max, 8 * cap);
                    seen = realloc(seen, cap);
                }
                ht[h].k = kv; ht[h].b = b; ht[h].gid = ng;
                a->gkey[ng] = kv; a->bucket[ng] = b; a->count[ng] = 0; a->sum[ng] = 0.0; a->min[ng] = INFINITY; a->max[ng] = -INFINITY; seen[ng] = 0;
                ng++;
            }
            cur_g = ht[h].gid; cur_k = kv; cur_b = b;
        }
        a->count[cur_g]++;
        if (value_col >= 0 && t->valid[value_col][row]) {
            double v = slot_to_double(t->vals[value_col][row], types[value_col]);
            a->sum[cur_g] += v;
            if (!seen[cur_g] || v < a->min[cur_g]) a->min[cur_g] = v;
            if (!seen[cur_g] || v > a->max[cur_g]) a->max[cur_g] = v;
            seen[cur_g] = 1;
        }
    }
    /* emit sorted by (group value, bucket) */
    int64_t *ord = malloc(8 * (ng ? ng : 1));
    for (int64_t i = 0; i < ng; i++) ord[i] = i;
    g_sort_type = group_col >= 0 ? types[group_col] : OT_U64; g_sort_res = a;
    qsort(ord, (size_t)ng, sizeof(int64_t), cmp_group_ids);
    orc_agg_result *o = calloc(1, sizeof *o);
    int64_t oc = ng ? ng : 1;
    o->gkey = malloc(8 * oc); o->bucket = malloc(8 * oc); o->count = malloc(8 * oc); o->sum = malloc(8 * oc); o->min = malloc(8 * oc); o->max = malloc(8 * oc);
    for (int64_t i = 0; i < ng; i++) {
        int64_t g = ord[i];
        o->gkey[i] = a->gkey[g]; o->bucket[i] = a->bucket[g]; o->count[i] = a->count[g]; o->sum[i] = a->sum[g]; o->min[i] = a->min[g]; o->max[i] = a->max[g];
    }
    o->ngroups = ng;
    o->rows_in_files = stats[0]; o->rows_decoded = stats[1]; o->rows_filtered = stats[2]; o->rows_merged = stats[3]; o->rows_out = ns;
    free(ord); free(ht); free(seen); orc_agg_result_free(a);
    for (int i = 0; i < k; i++) { orc_table_free(st[i].t); free(st[i].chunk_end); }
    free(st); free(surv);
    *out = o; return 0;
}

/* S8: Timestamp::truncate_by (types.rs:82-85) */
int64_t orc_truncate_by(int64_t ts, int64_t duration_ms) { return ts / duration_ms * duration_ms; }

int orc_num_threads(void) { long n = sysconf(_SC_NPROCESSORS_ONLN); return n > 0 ? (int)n : 1; }
