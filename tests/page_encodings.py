"""TEST INFRASTRUCTURE: rewrite what is inside a Parquet file's pages the way other writers lay it out.

recode(data, encode) takes a file pyarrow wrote with PLAIN values, no dictionary and no compression (V1 or V2 data pages), parses every
column chunk's definition levels and values, and lets encode(chunk) lay the chunk out again as a list of pages (Page): any split into
data pages, a dictionary page, and for every page its value encoding (PLAIN, DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY,
DELTA_BYTE_ARRAY, RLE_DICTIONARY / PLAIN_DICTIONARY indices) and its level bytes.  The byte-level encoders below make the choices the
Parquet spec allows and pyarrow never makes: DELTA block / miniblock geometries, widths wider than needed, junk in the unused widths and
the padding bits, 64-bit arithmetic on INT32 deltas, the same for the length runs of DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY pages;
RLE / bit-packed hybrid runs split anywhere, wide index widths, width 0.

The chunk statistics stay byte for byte (a chunk with null_count = 0 keeps it); page headers, ColumnMetaData.encodings, the sizes and the
offsets are rewritten with tests/page_recode.py's Thrift reader / writer (encoding_stats, which would describe the old pages, is
dropped).  Every call checks itself: the baseline layout (the source's own pages) gives back the input byte for byte, and pyarrow reads
the recoded file equal to the source unless the caller says pyarrow refuses the layout."""
import copy
import io
import random
from dataclasses import dataclass
from typing import Optional

import numpy as np
import pyarrow.parquet as pq

import page_recode as pr
from page_recode import T_I32, T_STRUCT, Struct

PLAIN, PLAIN_DICT, RLE, BIT_PACKED, DELTA, DLBA, DBA, RLE_DICT = 0, 2, 3, 4, 5, 6, 7, 8
INT32, INT64, FLOAT, DOUBLE, BYTE_ARRAY = 1, 2, 4, 5, 6
_NP = {INT32: np.int32, INT64: np.int64, FLOAT: np.float32, DOUBLE: np.float64}
PH_DATA, PH_DICT, PH_V2_TYPE = 0, 2, 3
CM_ENCODINGS, CM_ENC_STATS = 2, 13


# ---- byte-level encoders

def uvarint(v):
    out = bytearray()
    while True:
        if v < 0x80:
            out.append(v)
            return bytes(out)
        out.append((v & 0x7F) | 0x80)
        v >>= 7


def zigzag(v):
    return 2 * v if v >= 0 else -2 * v - 1


def pack_bits(vals, w):
    """vals bit-packed LSB first, w bits each"""
    acc = 0
    for i, v in enumerate(vals):
        acc |= int(v) << (i * w)
    return acc.to_bytes((len(vals) * w + 7) // 8, "little")


def _wrap(v, bits):
    m = 1 << bits
    v %= m
    return v - m if v >= m >> 1 else v


def delta_encode(vals, bits, block=128, nmini=4, extra=0, junk=False, arith64=False, feats=None):
    """DELTA_BINARY_PACKED of the signed ints `vals` (physical width `bits`).  extra: bits added to every miniblock's width (capped at 64);
    junk: random bytes for the widths of the miniblocks past the last value and ones in the last miniblock's padding; arith64: the
    deltas of INT32 values taken in 64-bit arithmetic (widths up to 33, min delta outside i32) instead of wrapping in 32 bits."""
    feats = feats if feats is not None else {}
    per = block // nmini
    vals = [int(v) for v in vals]
    out = bytearray(uvarint(block) + uvarint(nmini) + uvarint(len(vals)) + uvarint(zigzag(vals[0] if vals else 0)))
    if len(uvarint(zigzag(vals[0] if vals else 0))) == 10:
        feats["varint_10_bytes"] = feats.get("varint_10_bytes", 0) + 1
    dbits = 64 if arith64 and bits == 32 else bits
    deltas = [_wrap(b - a, 64) if arith64 else _wrap(b - a, bits) for a, b in zip(vals, vals[1:])]
    rng = random.Random(len(vals) * 7 + block)
    for b0 in range(0, len(deltas), block):
        d = deltas[b0:b0 + block]
        mn = min(d)
        if not -(1 << 31) <= mn < 1 << 31 and bits == 32:
            feats["min_delta_outside_i32"] = feats.get("min_delta_outside_i32", 0) + 1
        if len(uvarint(zigzag(mn))) == 10:
            feats["varint_10_bytes"] = feats.get("varint_10_bytes", 0) + 1
        out += uvarint(zigzag(mn))
        adj = [(x - mn) % (1 << dbits) for x in d]
        widths, bodies = [], []
        for m in range(nmini):
            part = adj[m * per:(m + 1) * per]
            if not part:
                widths.append(rng.randrange(256) if junk else 0)
                if junk:
                    feats["junk_unused_width"] = feats.get("junk_unused_width", 0) + 1
                continue
            w = min(dbits, max(x.bit_length() for x in part) + extra)
            if w > 32 and bits == 32:
                feats["int32_width_over_32"] = feats.get("int32_width_over_32", 0) + 1
            if extra and w == 64:
                feats["width_64"] = feats.get("width_64", 0) + 1
            pad = per - len(part)
            if pad and junk and w:
                part = part + [(1 << w) - 1] * pad
                feats["ones_in_padding"] = feats.get("ones_in_padding", 0) + 1
            else:
                part = part + [0] * pad
            widths.append(w)
            bodies.append(pack_bits(part, w))
        out += bytes(widths) + b"".join(bodies)
    feats[f"delta_{block}_{nmini}"] = feats.get(f"delta_{block}_{nmini}", 0) + 1
    n = len(vals)
    for name, hit in (("count_0", n == 0), ("count_1", n == 1), ("count_block", n == block), ("count_block_plus_1", n == block + 1)):
        if hit:
            feats[name] = feats.get(name, 0) + 1
    return bytes(out)


def hybrid_encode(vals, w, style, feats=None, seed=0, pad=0):
    """RLE / bit-packed hybrid runs (no width byte, no length prefix) of `vals` at bit width w.  style:
    'rle'          only RLE runs: maximal runs of equal values (runs of 1 included)
    'packed'       only bit-packed runs, of 63, 1, 2, ... 62 groups in turn (the last group padded with zeros)
    'alternate'    RLE and bit-packed runs in turn, bit-packed ones over uniform stretches too
    'mod8'         RLE runs of 1..8 values between bit-packed runs, so that run ends fall at every position mod 8
    'short_rle'    RLE runs of 1, 1 and 2 values in turn, uniform stretches split too (1.5 bytes per value at width 1)
    'arrow'        Arrow's choice: RLE for runs of 8 or more, bit-packed groups otherwise
    pad: the value that fills the last bit-packed group (the spec does not say what it holds; writers use 0)"""
    feats = feats if feats is not None else {}
    vals = [int(v) for v in vals]
    nb = (w + 7) // 8
    out = bytearray()
    rng = random.Random(seed)

    def rle(v, n):
        out.extend(uvarint(n << 1) + int(v).to_bytes(nb, "little"))
        feats["rle_run"] = feats.get("rle_run", 0) + 1
        if n == 1:
            feats["rle_run_of_1"] = feats.get("rle_run_of_1", 0) + 1

    def packed(chunk):
        groups = (len(chunk) + 7) // 8
        assert 1 <= groups
        out.extend(uvarint((groups << 1) | 1) + pack_bits(chunk + [pad] * (groups * 8 - len(chunk)), w))
        if pad and len(chunk) % 8:
            feats["nonzero_padding"] = feats.get("nonzero_padding", 0) + 1
        feats["packed_run"] = feats.get("packed_run", 0) + 1
        if groups in (1, 63):
            feats[f"packed_groups_{groups}"] = feats.get(f"packed_groups_{groups}", 0) + 1
        if len(set(chunk)) == 1 and len(chunk) >= 8:
            feats["packed_uniform"] = feats.get("packed_uniform", 0) + 1

    def end(pos):
        feats[f"run_end_mod8_{pos % 8}"] = feats.get(f"run_end_mod8_{pos % 8}", 0) + 1

    i, n, k = 0, len(vals), 0
    if style == "rle":
        while i < n:
            j = i
            while j < n and vals[j] == vals[i]:
                j += 1
            rle(vals[i], j - i)
            i = j
            end(i)
    elif style == "short_rle":
        while i < n:
            j = i + 1
            while j < min(n, i + (1, 1, 2)[k % 3]) and vals[j] == vals[i]:
                j += 1
            k += 1
            rle(vals[i], j - i)
            i = j
            end(i)
    elif style == "packed":
        while i < n:
            g = (k + 62) % 63 + 1                      # 63 groups first, then 1, 2, ...
            k += 1
            packed(vals[i:i + 8 * g])
            i += 8 * g
            end(min(i, n))
    elif style in ("alternate", "mod8"):
        while i < n:
            if k % 2 == 0:
                m = (k // 2) % 8 + 1 if style == "mod8" else rng.randrange(1, 40)
                m = min(m, n - i)
                if style == "alternate" or len(set(vals[i:i + m])) == 1:
                    j = i
                    while j < i + m and vals[j] == vals[i]:
                        j += 1
                    rle(vals[i], j - i)
                    i = j
                else:
                    rle(vals[i], 1)
                    i += 1
            else:
                g = rng.randrange(1, 6)
                packed(vals[i:i + 8 * g])
                i = min(n, i + 8 * g)
            k += 1
            end(i)
    elif style == "arrow":
        while i < n:
            j = i
            while j < n and vals[j] == vals[i]:
                j += 1
            if j - i >= 8:
                rle(vals[i], j - i)
                i = j
            else:
                packed(vals[i:i + 8])
                i = min(n, i + 8)
    else:
        raise ValueError(style)
    return bytes(out)


def dlba_encode(vals, feats=None, **delta):
    """DELTA_LENGTH_BYTE_ARRAY of the byte strings `vals`: their lengths as DELTA_BINARY_PACKED (delta_encode's options), then the bytes"""
    feats = feats if feats is not None else {}
    feats["dlba_page"] = feats.get("dlba_page", 0) + 1
    return delta_encode([len(v) for v in vals], 32, feats=feats, **delta) + b"".join(vals)


def dba_encode(vals, feats=None, **delta):
    """DELTA_BYTE_ARRAY: the prefix each value shares with the one before it and the suffix lengths, both DELTA_BINARY_PACKED, then the
    suffixes"""
    feats = feats if feats is not None else {}
    feats["dba_page"] = feats.get("dba_page", 0) + 1
    pre, prev = [], b""
    for v in vals:
        k = 0
        while k < min(len(v), len(prev)) and v[k] == prev[k]:
            k += 1
        pre.append(k)
        prev = v
    if any(pre):
        feats["dba_shared_prefix"] = feats.get("dba_shared_prefix", 0) + 1
    return (delta_encode(pre, 32, feats=feats, **delta) + delta_encode([len(v) - k for v, k in zip(vals, pre)], 32, feats=feats, **delta)
            + b"".join(v[k:] for v, k in zip(vals, pre)))


# ---- the chunk model

@dataclass
class Chunk:
    """one column chunk as the source holds it"""
    ci: int
    name: str
    phys: int
    optional: bool
    levels: np.ndarray                 # uint8 [num_rows]: 1 = a value
    values: list                       # the non-null values: python ints / floats' bit patterns as ints, or bytes
    width: int                         # PLAIN bytes of a fixed-width value (0: BYTE_ARRAY)
    v2: bool
    src_pages: list                    # [(header Struct, levels bytes, values bytes)] of the source's data pages
    null_count_zero: bool


@dataclass
class Page:
    rows: int                          # rows of the page (levels)
    values: bytes                      # the encoded values
    encoding: int = PLAIN
    levels: Optional[bytes] = None     # RLE-hybrid bytes of the levels (no length prefix); None: the levels of the rows in Arrow's layout
    level_encoding: int = RLE
    dictionary: bool = False           # a dictionary page (rows = entries)
    v2: Optional[bool] = None          # None: the source's page version
    header: Optional[Struct] = None    # the source header to keep (the baseline)
    named: bool = True                 # a dictionary page: dictionary_page_offset names it (else it sits at data_page_offset)


def plain(chunk, vals):
    if chunk.phys == BYTE_ARRAY:
        return b"".join(len(v).to_bytes(4, "little") + v for v in vals)
    return b"".join(int(v).to_bytes(chunk.width, "little", signed=chunk.phys in (INT32, INT64) and int(v) < 0) for v in vals)


def signed(chunk, vals):
    """the values as the signed ints their physical type holds"""
    return [_wrap(int(v), 32 if chunk.phys == INT32 else 64) for v in vals]


def _decode_levels(buf, n):
    out, p = [], 0
    while len(out) < n:
        h = 0
        sh = 0
        while True:
            b = buf[p]
            p += 1
            h |= (b & 0x7F) << sh
            sh += 7
            if not b & 0x80:
                break
        if h & 1:
            for g in range(h >> 1):
                out += [(buf[p] >> k) & 1 for k in range(8)]
                p += 1
        else:
            out += [buf[p] & 1] * (h >> 1)
            p += 1
    assert p == len(buf)
    return out[:n]


def _schema(fm):
    els = fm.get(2)[1][1:]
    return [(e.get(4).decode(), e.get(1), e.get(3)) for e in els]


def chunks_of(data):
    """[[Chunk per column] per row group] of a PLAIN, uncompressed, dictionary-free source"""
    fm, _ = pr.footer(data)
    cols = _schema(fm)
    res = []
    for rg in fm.get(pr.FM_ROW_GROUPS)[1]:
        row = []
        for ci, cc in enumerate(rg.get(pr.RG_COLUMNS)[1]):
            cm = cc.get(pr.CC_META)
            name, phys, rep = cols[ci]
            assert cm.get(pr.CM_CODEC) == pr.UNCOMPRESSED and not cm.has(pr.CM_DICT_OFF), "the source must be PLAIN and uncompressed"
            optional = rep == 1
            width = {INT32: 4, FLOAT: 4, INT64: 8, DOUBLE: 8, BYTE_ARRAY: 0}[phys]
            levels, values, src = [], [], []
            for ph, hpos, body in pr.chunk_pages(data, cm):
                assert ph.get(pr.PH_TYPE) in (PH_DATA, PH_V2_TYPE)
                payload = data[body:body + ph.get(pr.PH_CSIZE)]
                v2 = ph.get(pr.PH_V2)
                dh = v2 if v2 is not None else ph.get(5)
                nv = dh.get(1)
                assert dh.get(4 if v2 is not None else 2) == PLAIN
                if v2 is not None:
                    lv = payload[:v2.get(pr.V2_DEF_LEN, 0)]
                    vb = payload[len(lv):]
                elif optional:
                    ln = int.from_bytes(payload[:4], "little")
                    lv, vb = payload[4:4 + ln], payload[4 + ln:]
                else:
                    lv, vb = b"", payload
                lev = _decode_levels(lv, nv) if optional else [1] * nv
                nn = sum(lev)
                if phys == BYTE_ARRAY:
                    p, vals = 0, []
                    for _ in range(nn):
                        ln = int.from_bytes(vb[p:p + 4], "little")
                        vals.append(bytes(vb[p + 4:p + 4 + ln]))
                        p += 4 + ln
                    assert p == len(vb)
                else:
                    assert len(vb) == nn * width
                    vals = [int.from_bytes(vb[k * width:(k + 1) * width], "little") for k in range(nn)]
                levels += lev
                values += vals
                src.append((ph, bytes(lv), bytes(vb)))
            st = cm.get(12)
            row.append(Chunk(ci, name, phys, optional, np.array(levels, np.uint8), values, width, src[0][0].get(pr.PH_V2) is not None, src,
                             st is not None and st.get(3) == 0))
        res.append(row)
    return res


def baseline(chunk):
    """the source's own pages"""
    return [Page(rows=ph.get(pr.PH_V2).get(1) if ph.get(pr.PH_V2) is not None else ph.get(5).get(1), values=vb, levels=lv, header=ph)
            for ph, lv, vb in chunk.src_pages]


def split_rows(chunk, sizes):
    """row ranges of pages of the given sizes (the last size repeats), covering the chunk"""
    n, i, k, out = len(chunk.levels), 0, 0, []
    while i < n:
        s = sizes[min(k, len(sizes) - 1)]
        out.append((i, min(n, i + s)))
        i += s
        k += 1
    return out


def values_in(chunk, a, b):
    """the non-null values of rows [a, b)"""
    lo = int(chunk.levels[:a].sum())
    return chunk.values[lo:lo + int(chunk.levels[a:b].sum())]


def bit_packed_levels(levels):
    """deprecated BIT_PACKED levels at width 1: MSB first, no length"""
    out = bytearray((len(levels) + 7) // 8)
    for i, v in enumerate(levels):
        out[i // 8] |= int(v) << (7 - i % 8)
    return bytes(out)


# ---- the rewrite

def _data_header(page, usize, csize, v2):
    if page.header is not None:
        ph = copy.deepcopy(page.header)
    elif v2:
        ph = Struct([[1, T_I32, PH_V2_TYPE], [2, T_I32, 0], [3, T_I32, 0],
                     [8, T_STRUCT, Struct([[1, T_I32, 0], [2, T_I32, 0], [3, T_I32, 0], [4, T_I32, 0], [5, T_I32, 0], [6, T_I32, 0]])]])
    else:
        ph = Struct([[1, T_I32, PH_DATA], [2, T_I32, 0], [3, T_I32, 0],
                     [5, T_STRUCT, Struct([[1, T_I32, 0], [2, T_I32, 0], [3, T_I32, RLE], [4, T_I32, RLE]])]])
    ph.set(pr.PH_USIZE, usize)
    ph.set(pr.PH_CSIZE, csize)
    return ph


def _page_bytes(chunk, page, template_v2, nonnull):
    """(header, payload) of one page; nonnull: its rows that hold a value"""
    if page.dictionary:
        ph = Struct([[1, T_I32, PH_DICT], [2, T_I32, len(page.values)], [3, T_I32, len(page.values)],
                     [7, T_STRUCT, Struct([[1, T_I32, page.rows], [2, T_I32, page.encoding]])]])
        return pr.write_struct(ph), page.values
    v2 = template_v2 if page.v2 is None else page.v2
    lv = page.levels if page.levels is not None else b""
    if v2:
        payload = lv + page.values
        ph = _data_header(page, len(payload), len(payload), True)
        h = ph.get(pr.PH_V2)
        if page.header is None:
            h.set(1, page.rows)
            h.set(2, page.rows - nonnull)
            h.set(3, page.rows)
            h.set(4, page.encoding)
            h.set(5, len(lv))
            h.set(6, 0)
    else:
        if not chunk.optional:
            lv = b""
        elif page.level_encoding == RLE:
            lv = len(lv).to_bytes(4, "little") + lv
        payload = lv + page.values                     # (deprecated BIT_PACKED levels have no length in front)
        ph = _data_header(page, len(payload), len(payload), False)
        if page.header is None:
            h = ph.get(5)
            h.set(1, page.rows)
            h.set(2, page.encoding)
            h.set(3, page.level_encoding)
    return pr.write_struct(ph), payload


def recode(data, encode, pyarrow_reads=True, drop_stats=()):
    """`data` with every column chunk laid out by encode(chunk) -> [Page] (None: the baseline), checked as the module docstring says.
    drop_stats: the columns whose chunk statistics are removed too (no null_count: the engine plans a validity buffer for them)."""
    data = bytes(data)
    assert _rewrite(data, lambda c: None, ()) == data, "the baseline layout does not give back the input"
    out = _rewrite(data, encode, drop_stats)
    if pyarrow_reads:
        got = pq.read_table(io.BytesIO(out))
        assert got.equals(pq.read_table(io.BytesIO(data))), "pyarrow reads the recoded file differently"
    return out


def _rewrite(data, encode, drop_stats):
    fm, foot = pr.footer(data)
    all_chunks = chunks_of(data)
    out = bytearray(data[:4])
    for rg, chunks in zip(fm.get(pr.FM_ROW_GROUPS)[1], all_chunks):
        rg_dc = 0
        new_starts = []
        for cc, chunk in zip(rg.get(pr.RG_COLUMNS)[1], chunks):
            cm = cc.get(pr.CC_META)
            pages = encode(chunk)
            if pages is None:
                pages = baseline(chunk)
            start = len(out)
            new_starts.append(start)
            encs, lencs = set(), set()
            data_off = dict_off = None
            rows = 0
            for page in pages:
                nonnull = 0
                if not page.dictionary:
                    lv = chunk.levels[rows:rows + page.rows]
                    nonnull = int(lv.sum())
                    rows += page.rows
                    if page.levels is None and chunk.optional:
                        page.levels = hybrid_encode(lv, 1, "arrow")
                hdr, payload = _page_bytes(chunk, page, chunk.v2, nonnull)
                if page.dictionary:
                    dict_off = len(out)
                    encs.add(page.encoding)
                else:
                    if data_off is None:
                        data_off = len(out)
                    encs.add(page.encoding)
                    lencs.add(page.level_encoding)
                out += hdr + payload
            assert rows == len(chunk.levels), (chunk.name, rows, len(chunk.levels))
            new_tc = len(out) - start
            rg_dc += new_tc - cm.get(pr.CM_TOTAL_C)
            if not all(p.header is not None for p in pages):
                cm.set(CM_ENCODINGS, (T_I32, sorted(encs | lencs)))
                cm[:] = [f for f in cm if f[0] != CM_ENC_STATS]
            cm.set(pr.CM_TOTAL_C, new_tc)
            cm.set(pr.CM_TOTAL_U, new_tc)
            fields = [f for f in cm if f[0] != pr.CM_DICT_OFF]
            if dict_off is not None and pages[0].named:
                fields.append([pr.CM_DICT_OFF, pr.T_I64, dict_off])
            cm[:] = sorted(fields, key=lambda f: f[0])
            cm.set(pr.CM_DATA_OFF, start if dict_off is not None and not pages[0].named else data_off)
            if chunk.ci in drop_stats:
                cm[:] = [f for f in cm if f[0] != 12]
            if cc.has(pr.CC_FILE_OFFSET) and cc.get(pr.CC_FILE_OFFSET):
                cc.set(pr.CC_FILE_OFFSET, start)
        if rg.has(pr.RG_FILE_OFFSET) and new_starts:
            rg.set(pr.RG_FILE_OFFSET, new_starts[0])
        if rg.has(pr.RG_TOTAL_COMPRESSED):
            rg.set(pr.RG_TOTAL_COMPRESSED, rg.get(pr.RG_TOTAL_COMPRESSED) + rg_dc)
    meta = pr.write_struct(fm)
    return bytes(out) + meta + len(meta).to_bytes(4, "little") + b"PAR1"
