"""A model of Parquet split-block bloom filters written from the format specification alone (parquet-format BloomFilter.md), with a
Thrift-compact footer walk of its own: it shares no code with csrc/bloom.h or csrc/parquet_meta.cpp, so the tests can hold the library's
filters, probes and pruning against it.

  hash   xxHash64 (seed 0) of a value's PLAIN physical bytes: 4 for INT32 / FLOAT columns (1- and 2-byte integers widened to INT32),
         8 for INT64 / DOUBLE columns; NaN and signed zeros by their bits
  block  ((h >> 32) * num_blocks) >> 32, eight 32-bit words
  bits   word i gets 1 << ((uint32(h) * SALT[i]) >> 27)"""
import struct

import numpy as np
import pyarrow as pa

P1, P2, P3, P4, P5 = (0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5)
SALT = np.array([0x47b6137b, 0x44974d91, 0x8824ad5b, 0xa2b7289d, 0x705495c7, 0x2df1424b, 0x9efc4947, 0x5c6bfb31], dtype=np.uint32)
M64 = (1 << 64) - 1


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def xxh64(data: bytes, seed: int = 0) -> int:
    """xxHash64 of any byte string, scalar and unoptimised (the reference point of the vectorised 4- / 8-byte forms below)."""
    n, i = len(data), 0

    def rnd(acc, lane):
        return (_rotl((acc + lane * P2) & M64, 31) * P1) & M64

    if n >= 32:
        v = [(seed + P1 + P2) & M64, (seed + P2) & M64, seed, (seed - P1) & M64]
        while i + 32 <= n:
            for k in range(4):
                v[k] = rnd(v[k], struct.unpack_from("<Q", data, i + 8 * k)[0])
            i += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M64
        for k in range(4):
            h = (((h ^ rnd(0, v[k])) * P1) + P4) & M64
    else:
        h = (seed + P5) & M64
    h = (h + n) & M64
    while i + 8 <= n:
        h = ((_rotl(h ^ rnd(0, struct.unpack_from("<Q", data, i)[0]), 27) * P1) + P4) & M64
        i += 8
    if i + 4 <= n:
        h = ((_rotl(h ^ ((struct.unpack_from("<I", data, i)[0] * P1) & M64), 23) * P2) + P3) & M64
        i += 4
    while i < n:
        h = (_rotl(h ^ ((data[i] * P5) & M64), 11) * P1) & M64
        i += 1
    h ^= h >> 33
    h = (h * P2) & M64
    h ^= h >> 29
    h = (h * P3) & M64
    h ^= h >> 32
    return h


def _u64(x):
    return np.uint64(x)


def _vrotl(x, r):
    return (x << _u64(r)) | (x >> _u64(64 - r))


def _vaval(h):
    h = h ^ (h >> _u64(33))
    h = h * _u64(P2)
    h = h ^ (h >> _u64(29))
    h = h * _u64(P3)
    return h ^ (h >> _u64(32))


def hash_phys(phys: np.ndarray) -> np.ndarray:
    """Vectorised xxHash64 of PLAIN physical values: a uint32 array hashes 4 bytes each, a uint64 array 8 bytes each."""
    with np.errstate(over="ignore"):
        if phys.dtype == np.uint32:
            h = np.full(phys.shape, (P5 + 4) & M64, dtype=np.uint64)
            h ^= phys.astype(np.uint64) * _u64(P1)
            h = _vrotl(h, 23) * _u64(P2) + _u64(P3)
        else:
            x = phys.astype(np.uint64)
            h = np.full(phys.shape, (P5 + 8) & M64, dtype=np.uint64)
            h ^= _vrotl(x * _u64(P2), 31) * _u64(P1)
            h = _vrotl(h, 27) * _u64(P1) + _u64(P4)
        return _vaval(h)


def phys_values(arr) -> np.ndarray:
    """The PLAIN physical values of the non-null entries of an Arrow array (uint32 for INT32 / FLOAT columns, uint64 otherwise)."""
    arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
    arr = arr.drop_null()
    t = arr.type
    v = arr.to_numpy(zero_copy_only=False)
    if t in (pa.uint64(), pa.int64(), pa.float64()):
        return v.view(np.uint64) if v.dtype.itemsize == 8 else v.astype(np.uint64)
    if t == pa.float32():
        return v.view(np.uint32)
    return v.astype(np.int64).astype(np.uint32) if pa.types.is_signed_integer(t) else v.astype(np.uint32)


def build(phys: np.ndarray, num_bytes: int) -> bytes:
    """The bitset a writer produces for these physical values."""
    nblocks = num_bytes // 32
    words = np.zeros((nblocks, 8), dtype=np.uint32)
    if len(phys):
        h = hash_phys(phys)
        blk = ((h >> _u64(32)) * _u64(nblocks)) >> _u64(32)
        key = (h & _u64(0xffffffff)).astype(np.uint32)
        with np.errstate(over="ignore"):
            bits = np.left_shift(np.uint32(1), (key[:, None] * SALT[None, :]) >> np.uint32(27))
        np.bitwise_or.at(words, blk.astype(np.int64), bits)
    return words.astype("<u4").tobytes()


def may_contain(bitset: bytes, h: int) -> bool:
    nblocks = len(bitset) // 32
    b = ((h >> 32) * nblocks) >> 32
    words = struct.unpack_from("<8I", bitset, b * 32)
    key = h & 0xffffffff
    return all(words[i] & (1 << (((key * int(SALT[i])) & 0xffffffff) >> 27)) for i in range(8))


# ---------------------------------------------------------------------------------------------- the literals a planner may probe with
_INT_RANGE = {pa.uint8(): (0, 255), pa.uint16(): (0, 65535), pa.uint32(): (0, 2**32 - 1), pa.int8(): (-128, 127),
              pa.int16(): (-32768, 32767), pa.int32(): (-2**31, 2**31 - 1), pa.uint64(): (0, 2**64 - 1), pa.int64(): (-2**63, 2**63 - 1)}


def literal_hash(lit, t):
    """The hash of a literal as a column of Arrow type t stores it, or None when the column cannot represent it exactly
    (out of range, a float that does not round-trip through f32, NaN): such a predicate is never probed."""
    if pa.types.is_floating(t):
        d = float(lit)
        if d != d:
            return None
        if t == pa.float64():
            return int(hash_phys(np.array([d]).view(np.uint64))[0])
        f = np.float32(d)
        if np.array([float(f)]).view(np.uint64)[0] != np.array([d]).view(np.uint64)[0]:
            return None
        return int(hash_phys(np.array([f]).view(np.uint32))[0])
    lo, hi = _INT_RANGE[t]
    if not isinstance(lit, int) or not lo <= lit <= hi:
        return None
    if t in (pa.uint64(), pa.int64()):
        return int(hash_phys(np.array([lit & M64], dtype=np.uint64))[0])
    return int(hash_phys(np.array([lit & 0xffffffff], dtype=np.uint32))[0])


def bloom_keeps(bitset: bytes, t, op: str, lit) -> bool:
    """May a row group whose chunk has this filter match `col <op> lit`?  `=` / `in` only; any unrepresentable literal leaves the
    predicate to statistics."""
    if op not in ("eq", "in"):
        return True
    lits = list(lit) if op == "in" else [lit]
    hs = [literal_hash(x, t) for x in lits]
    if not hs or any(h is None for h in hs):
        return True
    return any(may_contain(bitset, h) for h in hs)


# ---------------------------------------------------------------------------------------------- a footer walk of its own
class _Thrift:
    def __init__(self, buf, pos):
        self.b, self.p = buf, pos

    def uvar(self):
        v, s = 0, 0
        while True:
            c = self.b[self.p]
            self.p += 1
            v |= (c & 0x7f) << s
            s += 7
            if not c & 0x80:
                return v

    def svar(self):
        v = self.uvar()
        return (v >> 1) ^ -(v & 1)

    def fields(self):
        fid = 0
        while True:
            h = self.b[self.p]
            self.p += 1
            if h == 0:
                return
            d, t = h >> 4, h & 15
            fid = fid + d if d else self.svar()
            yield fid, t

    def skip(self, t):
        if t in (1, 2):
            return
        if t == 3:
            self.p += 1
        elif t in (4, 5, 6):
            self.uvar()
        elif t == 7:
            self.p += 8
        elif t == 8:
            n = self.uvar()
            self.p += n
        elif t in (9, 10):
            for et in self.elems():
                self.skip(et) if et not in (1, 2) else setattr(self, "p", self.p + 1)
        elif t == 12:
            for _, t2 in self.fields():
                self.skip(t2)
        else:
            raise ValueError("thrift type %d" % t)

    def elems(self):
        h = self.b[self.p]
        self.p += 1
        n, et = h >> 4, h & 15
        if n == 15:
            n = self.uvar()
        for _ in range(n):
            yield et


def footer_blooms(data: bytes):
    """{(row group, column): dict(offset, length, offset_at, length_at)} from ColumnMetaData fields 14 / 15; *_at = the
    (start, end) byte range of the field's varint in the file, for tests that damage it."""
    flen = struct.unpack_from("<I", data, len(data) - 8)[0]
    t = _Thrift(data, len(data) - 8 - flen)
    out = {}
    for fid, ft in t.fields():
        if fid != 4:
            t.skip(ft)
            continue
        for g, _ in enumerate(t.elems()):
            for f2, t2 in t.fields():
                if f2 != 1:
                    t.skip(t2)
                    continue
                for c, _ in enumerate(t.elems()):
                    ent = {"offset": -1, "length": -1}
                    for f3, t3 in t.fields():
                        if f3 != 3:
                            t.skip(t3)
                            continue
                        for f4, t4 in t.fields():
                            if f4 in (14, 15):
                                a = t.p
                                v = t.svar()
                                key = "offset" if f4 == 14 else "length"
                                ent[key], ent[key + "_at"] = v, (a, t.p)
                            else:
                                t.skip(t4)
                    out[(g, c)] = ent
    return out


def read_filter(data: bytes, offset: int):
    """(numBytes, header length, bitset) of the BloomFilterHeader at `offset`; the algorithm / hash / compression must be the spec's
    BLOCK / XXHASH / UNCOMPRESSED."""
    t = _Thrift(data, offset)
    nbytes, unions = None, set()
    for fid, ft in t.fields():
        if fid == 1:
            nbytes = t.svar()
        elif fid in (2, 3, 4):
            members = [f2 for f2, t2 in t.fields() if t.skip(t2) is None]
            assert members == [1], (fid, members)
            unions.add(fid)
        else:
            t.skip(ft)
    assert unions == {2, 3, 4} and nbytes is not None
    hlen = t.p - offset
    return nbytes, hlen, bytes(data[t.p:t.p + nbytes])
