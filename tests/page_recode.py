"""TEST INFRASTRUCTURE: rewrite a Parquet file's pages with another compressor.

recode(data, compress, codec) returns the file with every page's payload (dictionary and data pages, V1 and V2) replaced by
compress(page_bytes, column, page_no) — page_bytes the page's decompressed payload (a V2 page: the part after its levels, which stay
uncompressed), page_no the page's index in its column chunk — and the chunks' codec set to `codec` (a Parquet CompressionCodec number,
None: keep it).  Page headers and the footer go through a small generic Thrift compact-protocol reader / writer that keeps every field
it does not change, in order: sizes and offsets are updated (compressed_page_size; ColumnMetaData.codec, total_compressed_size,
total_uncompressed_size, data_page_offset, dictionary_page_offset; RowGroup sizes and offsets; the footer length), the key-value
metadata (the SST's schema) is kept byte for byte.  Page CRCs, page indexes and bloom filters are refused rather than half rewritten.

Every call checks itself: the identity compressor (each page's own stream) gives back the input byte for byte, pyarrow reads the recoded
file equal to the input, and every recoded page decompresses with pyarrow's codec (libsnappy / libzstd) to the source page's bytes."""
import io

import pyarrow as pa
import pyarrow.parquet as pq

UNCOMPRESSED, SNAPPY, ZSTD = 0, 1, 6
_CODEC_NAME = {SNAPPY: "snappy", ZSTD: "zstd"}

# compact protocol types
T_TRUE, T_FALSE, T_BYTE, T_I16, T_I32, T_I64, T_DOUBLE, T_BINARY, T_LIST, T_SET, T_MAP, T_STRUCT = range(1, 13)


class Struct(list):
    """A Thrift struct as its fields in wire order: [field id, type, value]; booleans keep their type (T_TRUE / T_FALSE)."""

    def get(self, fid, default=None):
        for f in self:
            if f[0] == fid:
                return f[2]
        return default

    def set(self, fid, value):
        for f in self:
            if f[0] == fid:
                f[2] = value
                return
        raise KeyError(fid)

    def has(self, fid):
        return any(f[0] == fid for f in self)


class _Reader:
    def __init__(self, buf, pos=0):
        self.b, self.p = buf, pos

    def varint(self):
        v = sh = 0
        while True:
            x = self.b[self.p]
            self.p += 1
            v |= (x & 0x7F) << sh
            sh += 7
            if not x & 0x80:
                return v

    def zigzag(self):
        v = self.varint()
        return (v >> 1) ^ -(v & 1)

    def value(self, t):
        if t in (T_TRUE, T_FALSE):
            return t == T_TRUE
        if t == T_BYTE:
            self.p += 1
            return self.b[self.p - 1]
        if t in (T_I16, T_I32, T_I64):
            return self.zigzag()
        if t == T_DOUBLE:
            self.p += 8
            return bytes(self.b[self.p - 8:self.p])
        if t == T_BINARY:
            n = self.varint()
            self.p += n
            return bytes(self.b[self.p - n:self.p])
        if t in (T_LIST, T_SET):
            h = self.b[self.p]
            self.p += 1
            n, et = h >> 4, h & 0x0F
            if n == 15:
                n = self.varint()
            if et in (T_TRUE, T_FALSE):
                vals = []
                for _ in range(n):
                    vals.append(self.b[self.p] == T_TRUE)
                    self.p += 1
                return (et, vals)
            return (et, [self.value(et) for _ in range(n)])
        if t == T_MAP:
            n = self.varint()
            if n == 0:
                return (0, [])
            kv = self.b[self.p]
            self.p += 1
            return (kv, [(self.value(kv >> 4), self.value(kv & 0x0F)) for _ in range(n)])
        if t == T_STRUCT:
            return self.struct()
        raise ValueError(f"thrift type {t}")

    def struct(self):
        s, last = Struct(), 0
        while True:
            h = self.b[self.p]
            self.p += 1
            if h == 0:
                return s
            t, d = h & 0x0F, h >> 4
            fid = last + d if d else self.zigzag()
            s.append([fid, t, self.value(t)])
            last = fid


class _Writer:
    def __init__(self):
        self.b = bytearray()

    def varint(self, v):
        while True:
            if v < 0x80:
                self.b.append(v)
                return
            self.b.append((v & 0x7F) | 0x80)
            v >>= 7

    def zigzag(self, v):
        self.varint((v << 1) ^ (v >> 63))

    def value(self, t, v):
        if t in (T_TRUE, T_FALSE):
            return
        if t == T_BYTE:
            self.b.append(v & 0xFF)
        elif t in (T_I16, T_I32, T_I64):
            self.zigzag(v)
        elif t == T_DOUBLE:
            self.b += v
        elif t == T_BINARY:
            self.varint(len(v))
            self.b += v
        elif t in (T_LIST, T_SET):
            et, vals = v
            if len(vals) < 15:
                self.b.append((len(vals) << 4) | et)
            else:
                self.b.append(0xF0 | et)
                self.varint(len(vals))
            for x in vals:
                if et in (T_TRUE, T_FALSE):
                    self.b.append(T_TRUE if x else T_FALSE)
                else:
                    self.value(et, x)
        elif t == T_MAP:
            kv, items = v
            self.varint(len(items))
            if items:
                self.b.append(kv)
                for k, x in items:
                    self.value(kv >> 4, k)
                    self.value(kv & 0x0F, x)
        elif t == T_STRUCT:
            self.struct(v)
        else:
            raise ValueError(f"thrift type {t}")

    def struct(self, s):
        last = 0
        for fid, t, v in s:
            if t in (T_TRUE, T_FALSE):
                t = T_TRUE if v else T_FALSE
            if 0 < fid - last <= 15:
                self.b.append(((fid - last) << 4) | t)
            else:
                self.b.append(t)
                self.zigzag(fid)
            self.value(t, v)
            last = fid
        self.b.append(0)


def read_struct(buf, pos=0):
    """-> (Struct, position after it)"""
    r = _Reader(buf, pos)
    s = r.struct()
    return s, r.p


def write_struct(s):
    w = _Writer()
    w.struct(s)
    return bytes(w.b)


# Parquet field ids (parquet.thrift)
PH_TYPE, PH_USIZE, PH_CSIZE, PH_CRC, PH_V2 = 1, 2, 3, 4, 8
V2_DEF_LEN, V2_REP_LEN, V2_IS_COMPRESSED = 5, 6, 7
FM_ROW_GROUPS = 4
RG_COLUMNS, RG_FILE_OFFSET, RG_TOTAL_COMPRESSED = 1, 5, 6
CC_FILE_OFFSET, CC_META = 2, 3
CC_INDEX_FIELDS = (4, 5, 6, 7)                                 # offset / column index offsets and lengths
CM_CODEC, CM_TOTAL_U, CM_TOTAL_C, CM_DATA_OFF, CM_INDEX_OFF, CM_DICT_OFF, CM_BLOOM_OFF = 4, 6, 7, 9, 10, 11, 14


def footer(data):
    """-> (FileMetaData, offset of the footer)"""
    assert data[:4] == b"PAR1" and data[-4:] == b"PAR1"
    n = int.from_bytes(data[-8:-4], "little")
    off = len(data) - 8 - n
    fm, end = read_struct(data, off)
    assert end == len(data) - 8
    return fm, off


def chunk_pages(data, cm):
    """the pages of column chunk `cm` (ColumnMetaData): [(header Struct, header offset, payload offset)]"""
    pos = cm.get(CM_DICT_OFF) or cm.get(CM_DATA_OFF)
    pos = min(pos, cm.get(CM_DATA_OFF))
    end = pos + cm.get(CM_TOTAL_C)
    pages = []
    while pos < end:
        ph, body = read_struct(data, pos)
        pages.append((ph, pos, body))
        pos = body + ph.get(PH_CSIZE)
    assert pos == end, "column chunk does not end at its last page"
    return pages


def _decompress(codec, buf, size):
    if codec == UNCOMPRESSED:
        assert len(buf) == size
        return bytes(buf)
    return pa.Codec(_CODEC_NAME[codec]).decompress(bytes(buf), decompressed_size=size, asbytes=True)


def _payload_parts(data, ph, body, codec):
    """(uncompressed levels prefix of a V2 page, the page's decompressed values part)"""
    v2 = ph.get(PH_V2)
    lv = v2.get(V2_DEF_LEN, 0) + v2.get(V2_REP_LEN, 0) if v2 is not None else 0
    comp = data[body + lv: body + ph.get(PH_CSIZE)]
    if v2 is not None and v2.get(V2_IS_COMPRESSED, True) is False:
        codec = UNCOMPRESSED
    return bytes(data[body:body + lv]), _decompress(codec, comp, ph.get(PH_USIZE) - lv)


def _rewrite(data, compress, codec):
    fm, foot = footer(data)
    out = bytearray(data[:4])
    old_pos = 4                                                # the chunks must tile the file from the magic to the footer
    for rg in fm.get(FM_ROW_GROUPS)[1]:
        rg_dc = 0
        new_starts = []
        for ci, cc in enumerate(rg.get(RG_COLUMNS)[1]):
            cm = cc.get(CC_META)
            if any(cc.has(f) for f in CC_INDEX_FIELDS) or cm.has(CM_INDEX_OFF) or cm.has(CM_BLOOM_OFF):
                raise ValueError("page indexes and bloom filters are not rewritten")
            src_codec = cm.get(CM_CODEC)
            dst_codec = src_codec if codec is None else codec
            pages = chunk_pages(data, cm)
            if pages[0][1] != old_pos:
                raise ValueError("bytes between column chunks")
            old_pos = pages[0][1] + cm.get(CM_TOTAL_C)
            start = len(out)
            new_starts.append(start)
            du = 0
            for pn, (ph, hpos, body) in enumerate(pages):
                if ph.has(PH_CRC):
                    raise ValueError("page CRCs are not rewritten")
                levels, raw = _payload_parts(data, ph, body, src_codec)
                payload = levels + bytes(compress(raw, ci, pn))
                v2 = ph.get(PH_V2)
                page_codec = dst_codec
                if v2 is not None and v2.get(V2_IS_COMPRESSED, True) is False and codec is None:
                    page_codec = UNCOMPRESSED                  # a V2 page stored uncompressed stays so unless the codec changes
                elif v2 is not None and v2.has(V2_IS_COMPRESSED):
                    v2.set(V2_IS_COMPRESSED, dst_codec != UNCOMPRESSED)
                if page_codec == UNCOMPRESSED:
                    assert payload == levels + raw
                else:                                          # a third-party decoder vouches for every stream
                    assert _decompress(page_codec, payload[len(levels):], len(raw)) == raw, (ci, pn)
                ph.set(PH_CSIZE, len(payload))
                hdr = write_struct(ph)
                if ph.get(PH_TYPE) == 2:
                    cm.set(CM_DICT_OFF, len(out))
                elif pn == 0 or pages[pn - 1][0].get(PH_TYPE) == 2:
                    cm.set(CM_DATA_OFF, len(out))
                out += hdr + payload
                du += len(hdr) - (body - hpos)                 # total_uncompressed_size counts the headers
            new_tc = len(out) - start
            rg_dc += new_tc - cm.get(CM_TOTAL_C)
            cm.set(CM_TOTAL_C, new_tc)
            cm.set(CM_TOTAL_U, cm.get(CM_TOTAL_U) + du)
            cm.set(CM_CODEC, dst_codec)
            if cc.has(CC_FILE_OFFSET) and cc.get(CC_FILE_OFFSET) not in (0, pages[0][1]):
                raise ValueError("ColumnChunk.file_offset is not the chunk's start")
            if cc.has(CC_FILE_OFFSET) and cc.get(CC_FILE_OFFSET):
                cc.set(CC_FILE_OFFSET, start)
        if rg.has(RG_FILE_OFFSET) and new_starts:
            rg.set(RG_FILE_OFFSET, new_starts[0])
        if rg.has(RG_TOTAL_COMPRESSED):
            rg.set(RG_TOTAL_COMPRESSED, rg.get(RG_TOTAL_COMPRESSED) + rg_dc)
    if old_pos != foot:
        raise ValueError("bytes between the last column chunk and the footer")
    meta = write_struct(fm)
    return bytes(out) + meta + len(meta).to_bytes(4, "little") + b"PAR1"


def identity(data):
    """the compressor that re-emits every page's own stream"""
    fm, _ = footer(data)
    streams = {}
    for gi, rg in enumerate(fm.get(FM_ROW_GROUPS)[1]):
        for ci, cc in enumerate(rg.get(RG_COLUMNS)[1]):
            for pn, (ph, hpos, body) in enumerate(chunk_pages(data, cc.get(CC_META))):
                v2 = ph.get(PH_V2)
                lv = v2.get(V2_DEF_LEN, 0) + v2.get(V2_REP_LEN, 0) if v2 is not None else 0
                streams.setdefault((ci, pn), []).append(bytes(data[body + lv:body + ph.get(PH_CSIZE)]))
    it = {k: iter(v) for k, v in streams.items()}
    return lambda raw, ci, pn: next(it[(ci, pn)])


def recode(data, compress, codec=None):
    """`data` with every page recompressed by compress(page_bytes, column, page_no), the codec set to `codec` (None: unchanged); checked
    as the module docstring says"""
    data = bytes(data)
    assert _rewrite(data, identity(data), None) == data, "the Thrift round trip does not give back the input"
    out = _rewrite(data, compress, codec)
    want = pq.read_table(io.BytesIO(data))
    got = pq.read_table(io.BytesIO(out))
    assert got.equals(want), "pyarrow reads the recoded file differently"
    assert pq.ParquetFile(io.BytesIO(out)).schema_arrow.metadata == pq.ParquetFile(io.BytesIO(data)).schema_arrow.metadata
    return out


def page_streams(data, column):
    """the payload (after a V2 page's levels) of every data page of `column`, in file order: [(stream, uncompressed size)]"""
    fm, _ = footer(data)
    res = []
    for rg in fm.get(FM_ROW_GROUPS)[1]:
        for ph, hpos, body in chunk_pages(data, rg.get(RG_COLUMNS)[1][column].get(CC_META)):
            if ph.get(PH_TYPE) == 2:
                continue
            v2 = ph.get(PH_V2)
            lv = v2.get(V2_DEF_LEN, 0) + v2.get(V2_REP_LEN, 0) if v2 is not None else 0
            res.append((bytes(data[body + lv:body + ph.get(PH_CSIZE)]), ph.get(PH_USIZE) - lv))
    return res
