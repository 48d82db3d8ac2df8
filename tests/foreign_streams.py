"""TEST INFRASTRUCTURE: Snappy and Zstandard streams in the element choices other encoders make (pure Python, seeded).

libsnappy cuts its input into independent 64 KiB blocks, ends a literal only at a block end or before a match, writes the narrowest
literal header and copy form that fits, and never emits a copy under 4 bytes; libzstd in one-shot mode writes one Single_Segment frame
with its content size.  The streams here are all valid and decode with libsnappy / libzstd, but make the other choices the formats allow:
copies across 64 KiB and with offsets of 65 536 or more, 1-3 byte copies, wide literal headers, literals split anywhere, streaming
frames without content size, several frames per page, skippable frames, checksums, raw / RLE blocks only.

Every encoder returns (stream, counts): what it emitted, so that a test can assert that the feature a case claims to exercise occurred."""
from collections import Counter

import numpy as np
import pyarrow as pa

BLOCK = 65536


class Stream:
    """A raw Snappy stream written element by element; `out` is what it decodes to, `counts` what was emitted.

    copy(kind=1 | 2 | 4) forces the element form (None: the narrowest that fits); lit(hdr=0..4) forces the number of literal length
    bytes after the tag (None: the narrowest)."""

    def __init__(self, seed=1):
        self.rng = np.random.default_rng(seed)
        self.body = bytearray()
        self.out = bytearray()
        self.counts = Counter()

    def lit(self, data, hdr=None):
        data = bytes(data)
        n = len(data) - 1
        assert n >= 0
        if hdr is None:
            hdr = 0 if n < 60 else (n.bit_length() + 7) // 8
        if hdr == 0:
            assert n < 60
            self.body.append(n << 2)
        else:
            assert n < 1 << (8 * hdr)
            self.body.append((59 + hdr) << 2)
            self.body += n.to_bytes(hdr, "little")
            if n < 60 or hdr > (n.bit_length() + 7) // 8:
                self.counts["wide_literal_header"] += 1
        start = len(self.out)
        self.body += data
        self.out += data
        self.counts["literal"] += 1
        end = len(self.out)
        if end % BLOCK and (end // BLOCK) != (start // BLOCK):
            self.counts["literal_across_64k"] += 1
        return self

    def rand(self, n):
        return self.lit(self.rng.integers(0, 256, n, dtype=np.uint8).tobytes())

    def copy(self, off, ln, check=True, kind=None):
        if kind is None:
            kind = 1 if 4 <= ln <= 11 and 0 < off < 2048 else (2 if off < 65536 else 4)
        if kind == 1:
            assert 4 <= ln <= 11 and off < 2048
            self.body += bytes([1 | ((ln - 4) << 2) | ((off >> 8) << 5), off & 0xFF])
        elif kind == 2:
            assert 1 <= ln <= 64 and off < 65536
            self.body += bytes([2 | ((ln - 1) << 2)]) + off.to_bytes(2, "little")
            if 4 <= ln <= 11 and off < 2048:
                self.counts["copy2_where_copy1_fits"] += 1
        else:
            assert 1 <= ln <= 64 and off < 1 << 32
            self.body += bytes([3 | ((ln - 1) << 2)]) + off.to_bytes(4, "little")
            if off >= 65536:
                self.counts["offset_over_64k"] += 1
        self.counts[f"copy{kind}"] += 1
        if ln < 4:
            self.counts["copy_under_4"] += 1
        if check:
            pos = len(self.out)
            assert 0 < off <= pos
            if (pos - off) // BLOCK != (pos + ln - 1) // BLOCK:
                self.counts["copy_across_64k"] += 1
            for _ in range(ln):
                self.out.append(self.out[-off])
        return self

    def pair(self, L, back):
        """a value of L literal bytes and 8 - L bytes of the value `back` values earlier (or the earliest one there is)"""
        back = min(back, (len(self.out) + L) // 8)
        return self.rand(L).copy(8 * back, 8 - L)

    def pairs(self, n, L=1, back=1):
        for i in range(n):
            self.pair(L if np.isscalar(L) else int(self.rng.choice(L)), back if np.isscalar(back) else int(self.rng.choice(back)))
        return self

    def bytes(self):
        n, head = len(self.out), bytearray()
        while True:
            head.append((n & 0x7F) | (0x80 if n > 0x7F else 0))
            n >>= 7
            if not n:
                return bytes(head + self.body)


def _matches(raw, window, min_len=4):
    """Greedy LZ77 parse of `raw` with a hash of 4-byte sequences over the last `window` bytes (the whole page when window is None):
    yields ("lit", start, end) and ("copy", offset, length) in order; a copy's length is unbounded (the caller cuts it)."""
    raw = bytes(raw)
    n, last, i, lit0 = len(raw), {}, 0, 0
    while i < n:
        best_len, best_off = 0, 0
        if i + 4 <= n:
            key = raw[i:i + 4]
            j = last.get(key)
            last[key] = i
            if j is not None and (window is None or i - j <= window):
                ln = 4
                while i + ln < n and raw[j + ln] == raw[i + ln]:
                    ln += 1
                best_len, best_off = ln, i - j
        if best_len >= min_len:
            if lit0 < i:
                yield ("lit", lit0, i)
            yield ("copy", best_off, best_len)
            for k in range(i + 1, min(i + best_len, n - 3)):
                last[raw[k:k + 4]] = k
            i += best_len
            lit0 = i
        else:
            i += 1
    if lit0 < n:
        yield ("lit", lit0, n)


def _emit_parse(s, raw, parse, kind=None, cut=None, lit_hdr=None):
    """writes a parse of _matches: copies as `kind` (None: the narrowest form) in pieces of `cut()` bytes (None: 64), literals with
    lit_hdr(length) length bytes (None: the narrowest)"""
    for e in parse:
        if e[0] == "lit":
            s.lit(raw[e[1]:e[2]], hdr=lit_hdr(e[2] - e[1]) if lit_hdr else None)
            continue
        _, off, ln = e
        while ln:
            form = None if kind == 1 and off >= 2048 else kind
            if form == 1:
                k = min(ln, 11)
                if 0 < ln - k < 4:
                    k = ln - 4
            else:
                k = min(ln, cut() if cut else 64)
            s.copy(off, k, kind=form)
            ln -= k


def _finish(s, raw):
    assert bytes(s.out) == bytes(raw)
    return s.bytes(), dict(s.counts)


def snappy_copy1_only(raw, seed=0):
    """every copy as a 1-byte-offset element where that form fits (4-11 bytes, offset < 2048): long matches become many short ones"""
    s = Stream(seed)
    _emit_parse(s, raw, _matches(raw, 2047), kind=1)
    return _finish(s, raw)


def snappy_copy2_only(raw, seed=0):
    """every copy as a 2-byte-offset element, also where a 1-byte-offset one fits; matches over the last 65 535 bytes"""
    s = Stream(seed)
    _emit_parse(s, raw, _matches(raw, 65535), kind=2)
    return _finish(s, raw)


def snappy_copy4_everywhere(raw, seed=0):
    """every copy as a 4-byte-offset element, short offsets included; matches over the whole page"""
    s = Stream(seed)
    _emit_parse(s, raw, _matches(raw, None), kind=4)
    return _finish(s, raw)


def snappy_one_window(raw, seed=0):
    """matches searched over the whole page: copies across every 64 KiB boundary, offsets above 65 535 on pages over 64 KiB, runs as
    chained 64-byte copies at small offsets"""
    s = Stream(seed)
    _emit_parse(s, raw, _matches(raw, None))
    return _finish(s, raw)


def snappy_short_copies(raw, seed=0):
    """matches cut into pieces of 1-3 bytes mixed with longer ones"""
    s = Stream(seed)
    rng = np.random.default_rng(seed)
    _emit_parse(s, raw, _matches(raw, 65535), kind=2, cut=lambda: int(rng.choice([1, 2, 3, 3, 8, 64])))
    return _finish(s, raw)


def snappy_wide_literal_headers(raw, seed=0):
    """every literal header with 1-4 length bytes, also where the tag alone would do"""
    s = Stream(seed)
    rng = np.random.default_rng(seed)
    _emit_parse(s, raw, _matches(raw, 65535), lit_hdr=lambda n: max((n - 1).bit_length() + 7 >> 3, int(rng.integers(1, 5))))
    return _finish(s, raw)


def snappy_random_parse(raw, seed=0):
    """at each position a seeded choice between a literal of random length and a copy from a random earlier occurrence of the next
    bytes (any distance, any length from 1 up to the match), so element boundaries fall anywhere"""
    raw = bytes(raw)
    rng = np.random.default_rng(seed)
    s = Stream(seed)
    where = {}
    i, n = 0, len(raw)
    while i < n:
        cands = where.get(raw[i:i + 2]) if i + 2 <= n else None
        if cands and rng.random() < 0.7:
            j = cands[int(rng.integers(0, len(cands)))]
            ln = 2
            while i + ln < n and ln < 64 and raw[j + ln] == raw[i + ln]:
                ln += 1
            ln = int(rng.integers(1, ln + 1))
            s.copy(i - j, ln, kind=None if ln >= 4 else (2 if i - j < 65536 else 4))
        else:
            ln = int(min(n - i, rng.choice([1, 2, 5, 17, 100, 3000])))
            s.lit(raw[i:i + ln])
        for k in range(i, min(i + ln, n - 1)):
            lst = where.setdefault(raw[k:k + 2], [])
            lst.append(k)
            if len(lst) > 8:
                lst.pop(int(rng.integers(0, 8)))
        i += ln
    return _finish(s, raw)


def snappy_literals_split(raw, points, hdr=None):
    """a literals-only stream of `raw` with a literal boundary at each byte position of `points` (positions inside (0, len))"""
    s = Stream(0)
    cuts = [0] + sorted(set(int(p) for p in points if 0 < p < len(raw))) + [len(raw)]
    for a, b in zip(cuts, cuts[1:]):
        s.lit(raw[a:b], hdr=hdr)
    return _finish(s, raw)


def snappy_lopsided(raw, front):
    """the first `front` bytes as one literal, whatever they hold, and the rest parsed for matches over the whole page: a stream whose
    front compresses far worse than its tail"""
    raw = bytes(raw)
    s = Stream(0)
    parse, pos = [], 0
    for e in _matches(raw, None):
        ln = e[2] - e[1] if e[0] == "lit" else e[2]
        if pos + ln > front:
            if pos >= front:
                parse.append(e)
            elif e[0] == "lit":                                   # an element across the cut: its part behind the cut
                parse.append(("lit", front, e[2]))
            else:
                parse.append(("copy", e[1], pos + ln - front))
        pos += ln
    if front:
        s.lit(raw[:front])
    _emit_parse(s, raw, parse)
    return _finish(s, raw)


SNAPPY_ENCODERS = {
    "copy1_only": snappy_copy1_only,
    "copy2_only": snappy_copy2_only,
    "copy4_everywhere": snappy_copy4_everywhere,
    "one_window": snappy_one_window,
    "short_copies": snappy_short_copies,
    "wide_literal_headers": snappy_wide_literal_headers,
    "random_parse": snappy_random_parse,
}


# ---- Zstandard

ZSTD_MAGIC = b"\x28\xb5\x2f\xfd"


def zstd_one_shot(raw, level=3):
    return pa.Codec("zstd", compression_level=level).compress(bytes(raw), asbytes=True)


def zstd_streaming(raw, flush_every=0):
    """one frame from libzstd's streaming API: Frame_Header_Descriptor 0x00 (a Window_Descriptor, no content size); a flush every
    `flush_every` bytes ends a block there"""
    sink = pa.BufferOutputStream()
    with pa.CompressedOutputStream(sink, "zstd") as out:
        raw = bytes(raw)
        step = flush_every or max(len(raw), 1)
        for i in range(0, len(raw), step):
            out.write(raw[i:i + step])
            if flush_every:
                out.flush()
    return sink.getvalue().to_pybytes()


def skippable_frame(payload, nibble=0):
    return (0x184D2A50 + nibble).to_bytes(4, "little") + len(payload).to_bytes(4, "little") + bytes(payload)


def zstd_with_checksum(raw, level=3):
    """a one-shot frame with the Content_Checksum_flag set and the low 32 bits of xxHash64(content) behind the last block"""
    from bloom_model import xxh64
    f = bytearray(zstd_one_shot(raw, level))
    assert f[:4] == ZSTD_MAGIC and not f[4] & 0x04
    f[4] |= 0x04
    return bytes(f) + (xxh64(bytes(raw)) & 0xFFFFFFFF).to_bytes(4, "little")


def zstd_raw_rle(raw, seed=0, window_descriptor=False):
    """a hand-built frame of raw and RLE blocks only (runs of one byte as RLE blocks), ending in an empty raw last block"""
    raw = bytes(raw)
    rng = np.random.default_rng(seed)
    if window_descriptor:
        out = bytearray(ZSTD_MAGIC + bytes([0x00, (7 << 3)]))          # no content size; window 2^(10 + 7) = 128 KiB
    else:
        out = bytearray(ZSTD_MAGIC + bytes([0xA0]) + len(raw).to_bytes(4, "little"))
    i = 0
    while i < len(raw):
        j = i
        while j < len(raw) and raw[j] == raw[i] and j - i < 131072:
            j += 1
        if j - i >= 8:
            out += (((j - i) << 3) | (1 << 1)).to_bytes(3, "little") + raw[i:i + 1]
            i = j
            continue
        k = i + int(rng.integers(1, 5000))
        k = min(k, len(raw))
        while k < len(raw) and k - i < 131072:                        # stop a raw block where a run starts
            if raw[k:k + 8] == raw[k:k + 1] * 8:
                break
            k += 1
        out += ((k - i) << 3).to_bytes(3, "little") + raw[i:k]
        i = k
    out += (1).to_bytes(3, "little")                                 # empty raw block, last
    return bytes(out)


def zstd_frames(raw, parts, level=3):
    """`parts` one-shot frames back to back, each holding a slice of raw"""
    raw = bytes(raw)
    cuts = [len(raw) * k // parts for k in range(parts + 1)]
    return b"".join(zstd_one_shot(raw[a:b], level) for a, b in zip(cuts, cuts[1:]))


def zstd_frame_header_bytes(stream):
    """the Frame_Header_Descriptor of every frame in the stream, skippable frames as the string "skip" (walks the frames with the
    blocks' sizes: raw / RLE / compressed)"""
    out, p = [], 0
    while p < len(stream):
        magic = int.from_bytes(stream[p:p + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            out.append("skip")
            p += 8 + int.from_bytes(stream[p + 4:p + 8], "little")
            continue
        assert stream[p:p + 4] == ZSTD_MAGIC
        fhd = stream[p + 4]
        out.append(fhd)
        p += 5 + (0 if fhd & 0x20 else 1) + [0, 1, 2, 4][fhd & 3] + [1 if fhd & 0x20 else 0, 2, 4, 8][fhd >> 6]
        while True:
            bh = int.from_bytes(stream[p:p + 3], "little")
            p += 3 + (1 if (bh >> 1) & 3 == 1 else bh >> 3)
            if bh & 1:
                break
        if fhd & 0x04:
            p += 4
    assert p == len(stream)
    return out


def _zstd_encoders():
    enc = {"stream": lambda r: zstd_streaming(r), "stream_flush_1k": lambda r: zstd_streaming(r, 1024),
           "stream_flush_7k": lambda r: zstd_streaming(r, 7 * 1024)}
    for lv in (-7, -1, 1, 3, 9, 19, 22):
        enc[f"level_{lv}"] = lambda r, lv=lv: zstd_one_shot(r, lv)
    enc["two_frames"] = lambda r: zstd_frames(r, 2)
    enc["three_frames"] = lambda r: zstd_frames(r, 3)
    enc["skippable_around"] = lambda r: skippable_frame(b"before", 3) + zstd_one_shot(r) + skippable_frame(b"", 15)
    enc["checksum"] = zstd_with_checksum
    enc["raw_rle"] = zstd_raw_rle
    enc["raw_rle_window"] = lambda r: zstd_raw_rle(r, window_descriptor=True)
    return enc


ZSTD_ENCODERS = _zstd_encoders()
