"""The gate decoder of the Snappy core (horaedb_b200/csrc/snappy_core.h: snappy_gate_page) on the CPU emulator
(tests/emu/snappy_gate_emu.cpp).

The decoder turns the Snappy stream of a 4-byte column page straight into one pass bit per value (the row-group gate of a gate-first
scan) without producing the page.  Every case here is checked against libsnappy's decoding of the same stream, tested on the host: the
bitmap, the last passing row, and whether the page was taken in the bit domain or handed back to be decoded the byte way (the result of
the byte way is the byte decoder's, tested by the other emulator files and by the GPU suite).  Streams: the benchmark's `tag` pages cut
from an `sstgen` SST, and exact element sequences written by the small Snappy writer of test_snappy_value_mode_emu.py.  Every case runs
with the lanes in order and in a pseudo-random order."""
import ctypes as C
import os
import subprocess

import numpy as np
import pyarrow as pa
import pytest

from test_emu_on_sst_pages import _pages
from test_snappy_value_mode_emu import Stream

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "snappy_gate_emu.cpp")
DEPS = [SRC, os.path.join(HERE, "..", "horaedb_b200", "csrc", "snappy_core.h"), os.path.join(HERE, "emu", "warp_emu.h")]
OUT = os.path.join(HERE, "emu", "_build", "libsnappy_gate_emu.so")
ORDERS = (0, 7)
PREDS = [(3, 0), (0, 0), (5, 7), (1000, 0), (0, 0xFFFFFFFF)]      # pass <=> value - lo <= span (u32): =, =, range, no match, all match


@pytest.fixture(scope="module")
def emu():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(p) for p in DEPS):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", OUT, SRC])
    lib = C.CDLL(OUT)
    lib.emu_gate_page.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                  C.POINTER(C.c_uint32), C.POINTER(C.c_long)]
    lib.emu_gate_page.restype = C.c_int
    lib.emu_set_order.argtypes = [C.c_int]
    return lib


def gate(lib, comp, ulen, optional, nrows, lo, span, order, flip=0):
    """-> (taken, bits as bools, last)"""
    lib.emu_set_order(order)
    bits = np.full((nrows + 31) // 32 + 1, 0xA5A5A5A5, dtype=np.uint32)
    last, n = C.c_uint32(0), C.c_long(0)
    r = lib.emu_gate_page(comp, len(comp), ulen, int(optional), nrows, flip, lo, span, bits.ctypes.data, C.byref(last), C.byref(n))
    lib.emu_set_order(0)
    assert r in (0, 1), r                                          # 0 / 1; anything else is an emulator error (a collective not all lanes reached)
    assert bits[-1] == 0xA5A5A5A5                                  # nothing written past the bitmap
    if not r:
        assert (bits == 0xA5A5A5A5).all()
        return False, None, None
    words = bits[:-1]
    got = np.unpackbits(words.view(np.uint8), bitorder="little").astype(bool)
    assert not got[nrows:].any()                                   # bits past the last row are zero
    return True, got[:nrows], last.value


def expect(raw, optional, lo, span, flip=0):
    raw = np.frombuffer(bytes(raw), dtype=np.uint8)
    start = 4 + int(raw[:4].view(np.uint32)[0]) if optional else 0
    vals = raw[start:].view(np.uint32)
    ok = ((vals ^ np.uint32(flip)) - np.uint32(lo)) <= np.uint32(span)
    return ok, (int(np.nonzero(ok)[0].max()) + 1 if ok.any() else 0)


def check(lib, comp, raw, optional=False, preds=PREDS, taken=True):
    nrows = (len(raw) - (4 + int.from_bytes(bytes(raw[:4]), "little") if optional else 0)) // 4
    for lo, span in preds:
        exp, last = expect(raw, optional, lo, span)
        for order in ORDERS:
            t, got, gl = gate(lib, comp, len(raw), optional, nrows, lo, span, order)
            assert t == taken
            if t:
                assert (got == exp).all(), (lo, span, np.nonzero(got != exp)[0][:8])
                assert gl == last


def bench_tag_pages():
    import bench
    from horaedb_b200 import sstgen
    data, _ = sstgen.synth_sst(0, 120, bench.POINTS, bench.DELTA_MS, seq=1, compression="snappy")
    codec = pa.Codec("snappy")
    for g, c, ptype, uncomp, payload in _pages(data):
        if c == 3 and ptype == 0:
            yield g, payload, codec.decompress(payload, uncomp, asbytes=True)


def test_bench_tag_pages_in_the_bit_domain(emu):
    """Every row group of a bench-shaped file (tag = series_id mod 16, 1 000 rows per series, nullable: a level prefix first): no page
    goes back to the byte decoder, and the bits match for =, a range, no match and all match."""
    n = 0
    for g, comp, raw in bench_tag_pages():
        check(emu, comp, raw, optional=True)
        n += 1
    assert n == 15


def _values(vals):
    return np.asarray(vals, dtype=np.uint32).tobytes()


def _level_prefix(k):
    """[u32 k][k level bytes]: a prefix of 4 + k bytes, so the values start at phase k mod 4"""
    return k.to_bytes(4, "little") + bytes(range(1, k + 1))


@pytest.mark.parametrize("k", range(0, 9))
def test_level_prefix_of_every_length(emu, k):
    rng = np.random.default_rng(k)
    vals = np.repeat(rng.integers(0, 6, 40), rng.integers(1, 40, 40))
    body = _level_prefix(k) + _values(vals)
    s = Stream(k).lit(body[:6])
    while len(s.out) < len(body):                                  # runs as copies of the value before, the rest literal
        i = len(s.out)
        if i >= 4 + k + 8 and body[i:i + 8] == body[i - 4:i + 4]:
            j = i
            while j < len(body) and j - i < 64 and body[j] == body[j - 4]:
                j += 1
            s.copy(4, j - i)
        else:
            s.lit(body[i:i + 1 + int(rng.integers(0, 6))])
    assert bytes(s.out) == body
    check(emu, s.bytes(), body, optional=True, preds=[(3, 0), (2, 2)])


@pytest.mark.parametrize("phase", range(4))
def test_mixed_values_at_every_phase(emu, phase):
    """Elements that end inside values: literals of 1..7 bytes and copies of 4..11 bytes from any offset, behind a first literal of
    16 + phase bytes."""
    rng = np.random.default_rng(10 + phase)
    s = Stream(phase).lit(rng.integers(0, 4, 16 + phase, dtype=np.uint8).tobytes())
    while len(s.out) < 1000:                                      # about 150 elements: within the table
        if rng.random() < 0.5:
            s.lit(rng.integers(0, 4, int(rng.integers(1, 8)), dtype=np.uint8).tobytes())
        else:
            s.copy(int(rng.integers(1, min(len(s.out), 200) + 1)), int(rng.integers(4, 12)))
    raw = bytes(s.out[:len(s.out) // 4 * 4])
    check(emu, _trimmed(s, len(raw)), raw, preds=[(1, 0), (0, 0x01010101), (2, 0)])


def _trimmed(s, n):
    """a stream of the first n output bytes of s: its elements up to n, the last one cut"""
    out = Stream()
    body, i = bytes(s.body), 0
    while len(out.out) < n:
        t = body[i]
        k = t & 3
        if k == 0:
            ln = (t >> 2) + 1
            out.lit(body[i + 1:i + 1 + min(ln, n - len(out.out))])
            i += 1 + ln
        else:
            if k == 1:
                ln, off, hl = ((t >> 2) & 7) + 4, ((t >> 5) << 8) | body[i + 1], 2
            elif k == 2:
                ln, off, hl = (t >> 2) + 1, int.from_bytes(body[i + 1:i + 3], "little"), 3
            else:
                ln, off, hl = (t >> 2) + 1, int.from_bytes(body[i + 1:i + 5], "little"), 5
            ln = min(ln, n - len(out.out))
            if ln < 4:
                out.lit(bytes(out.out[len(out.out) - off + j] if j < off else 0 for j in range(ln)))
                for j in range(ln):
                    out.out[-ln + j] = out.out[-ln + j - off]
                out.body[-ln:] = out.out[-ln:]
            else:
                out.copy(off, ln)
            i += hl
    assert bytes(out.out) == bytes(s.out[:n])
    return out.bytes()


@pytest.mark.parametrize("off", [1, 2, 3, 5, 6, 7])
def test_copies_that_are_not_value_aligned(emu, off):
    rng = np.random.default_rng(off)
    s = Stream(off).lit(rng.integers(0, 3, 12, dtype=np.uint8).tobytes())
    for _ in range(60):
        s.copy(off, int(rng.integers(4, 40)))
        s.lit(rng.integers(0, 3, int(rng.integers(1, 6)), dtype=np.uint8).tobytes())
    raw = bytes(s.out[:len(s.out) // 4 * 4])
    check(emu, _trimmed(s, len(raw)), raw, preds=[(0, 0), (1, 0x02020202), (0x00010000, 0)])


@pytest.mark.parametrize("period", [4, 8, 12])
def test_self_overlapping_copies(emu, period):
    """A run that repeats the last `period` bytes (run-length coding of a repeating sequence of values), long runs and short ones."""
    rng = np.random.default_rng(period)
    s = Stream(period)
    while len(s.out) < 20000:
        s.lit(_values(rng.integers(0, 5, period // 4)))
        for _ in range(int(rng.integers(1, 20))):
            s.copy(period, int(rng.integers(4, 65)))
    raw = bytes(s.out[:len(s.out) // 4 * 4])
    check(emu, _trimmed(s, len(raw)), raw)


def test_far_aligned_copies(emu):
    """Values copied from up to 32 KB back (the same tag some series earlier), out of the byte decoder's ring."""
    rng = np.random.default_rng(3)
    s = Stream(3)
    for _ in range(64):                                            # 4 KB of values in literals of 15 values
        s.lit(_values(rng.integers(0, 9, 15)))
    s.lit(_values([7]))
    while len(s.out) < 28 * 1024:                                  # a run of one value: one entry
        s.copy(4, 64)
    while len(s.out) < 32768 + 64:                                 # from the first 4 KB, 24-32 KB back
        s.copy(len(s.out) - 4 * int(rng.integers(0, 1000)), 4 * int(rng.integers(1, 17)))
        if rng.random() < 0.2:
            s.lit(_values(rng.integers(0, 9, 1)))
    raw = bytes(s.out[:8192 * 4])
    check(emu, _trimmed(s, len(raw)), raw)


def test_literals_of_every_short_length(emu):
    rng = np.random.default_rng(5)
    s = Stream(5)
    for ln in list(range(1, 61)) * 3:
        s.lit(rng.integers(0, 4, ln, dtype=np.uint8).tobytes())
    raw = bytes(s.out[:len(s.out) // 4 * 4])
    check(emu, _trimmed(s, len(raw)), raw, preds=[(0, 0), (0, 0x03030303)])


def test_what_the_bit_domain_declines(emu):
    """A long literal (an incompressible page), an element table over its 256 entries, a byte chase over its hop budget, a page with
    more rows than the bitmap holds, a level prefix whose length does not fill the page with values, a page size that is not the
    expected one: handed back untouched."""
    rng = np.random.default_rng(8)
    s = Stream(8).lit(rng.integers(0, 256, 400, dtype=np.uint8).tobytes())
    check(emu, s.bytes(), bytes(s.out), taken=False)
    s = Stream(8).lit(b"\1\0\0\0")                                 # 300 entries: literal, copy of another offset, ...
    for i in range(150):
        s.lit(bytes([i & 3, 0, 0, 0])).copy(4 * (1 + i % 3), 8)
    check(emu, s.bytes(), bytes(s.out), taken=False)
    s = Stream(8).lit(_values([1, 2]))                             # 100 short copies, each from the one or two before: every value mixed
    for i in range(100):
        s.copy(7 if i % 2 else 5, 4)
    raw = bytes(s.out[:len(s.out) // 4 * 4])
    check(emu, _trimmed(s, len(raw)), raw, taken=False)
    big = Stream(8).lit(_values([7]))
    while len(big.out) < 8193 * 4:
        big.copy(4, min(64, 8193 * 4 - len(big.out)))
    check(emu, big.bytes(), bytes(big.out), taken=False)
    body = _level_prefix(2) + _values(range(50))
    short = Stream(8).lit(body[:40]).lit(body[40:])
    nrows = (len(body) - 6) // 4
    for order in ORDERS:
        assert gate(emu, short.bytes(), len(body), True, nrows - 1, 0, 0, order)[0] is False
        assert gate(emu, short.bytes(), len(body) + 4, True, nrows, 0, 0, order)[0] is False


@pytest.mark.parametrize("cut", [1, 2, 5, 30])
def test_truncated_and_damaged_streams_are_declined(emu, cut):
    """The byte decoder reports these (errors 101-105); the bit path only declines them, so the result is the byte decoder's."""
    comp, raw = next((c, r) for g, c, r in bench_tag_pages() if g == 1)
    nrows = (len(raw) - 4 - int.from_bytes(raw[:4], "little")) // 4
    for order in ORDERS:
        assert gate(emu, comp[:-cut], len(raw), True, nrows, 3, 0, order)[0] is False
    bad = bytearray(comp)
    bad[3] = 2 | (3 << 2)                                          # a copy before the page's start
    bad[4:6] = (60000).to_bytes(2, "little")
    for order in ORDERS:
        assert gate(emu, bytes(bad), len(raw), True, nrows, 3, 0, order)[0] is False
