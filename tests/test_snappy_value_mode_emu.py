"""Value mode of the Snappy decoder (horaedb_b200/csrc/snappy_core.h) on the CPU emulator (tests/emu/snappy_value_emu.cpp).

Value mode decodes one (literal, copy) pair per 8-byte value, 32 values per warp step.  It is only an execution strategy: on any input the
output and the error codes are the decoder's without it.  The streams here are exact element sequences (a small Snappy writer below, so
shapes like 64 000-byte offsets or 5-byte copies are placed where the test wants them) and pyarrow-written Parquet pages (the benchmark's
timestamp column with its level prefix, a nullable column).  Every case runs in lane order 0 and in a random order, checks the bytes, and
asserts from the decoder's counters whether value mode took part."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import foreign_streams as fs
from foreign_streams import Stream

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "snappy_value_emu.cpp")
DEPS = [SRC, os.path.join(HERE, "..", "horaedb_b200", "csrc", "snappy_core.h"), os.path.join(HERE, "emu", "warp_emu.h")]
OUT = os.path.join(HERE, "emu", "_build", "libsnappy_emu_vm.so")
FIELDS = ("windows", "steps", "elements", "word_steps", "bytes", "parent_searches", "stage_hits", "value_steps")
ORDERS = (0, 7)          # lanes in order, and a pseudo-random order per interval between collectives


@pytest.fixture(scope="module")
def emu():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(p) for p in DEPS):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", OUT, SRC])
    lib = C.CDLL(OUT)
    lib.emu_snappy_page.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_long)]
    lib.emu_snappy_page.restype = C.c_int
    lib.emu_set_order.argtypes = [C.c_int]
    lib.emu_set_value_mode.argtypes = [C.c_int]
    return lib


def run(lib, comp, ulen, stop_at=0xFFFFFFFF, order=0, vmode=True):
    """-> (error code, output bytes, counters)"""
    lib.emu_set_order(order)
    lib.emu_set_value_mode(int(vmode))
    lib.emu_stats((C.c_long * len(FIELDS))())                    # reset
    out = np.full(ulen + 320, 0xEE, dtype=np.uint8)
    n = C.c_long(0)
    err = lib.emu_snappy_page(comp, len(comp), out.ctypes.data, ulen, stop_at, C.byref(n))
    st = (C.c_long * len(FIELDS))()
    lib.emu_stats(st)
    lib.emu_set_order(0)
    lib.emu_set_value_mode(1)
    assert (out[ulen + 64:] == 0xEE).all()                       # nothing written beyond the page's slack
    return err, out, dict(zip(FIELDS, st[:]))


def check(lib, comp, raw, value_mode, stop_at=0xFFFFFFFF):
    upto = min(len(raw), stop_at)
    for order in ORDERS:
        err, out, st = run(lib, comp, len(raw), stop_at, order)
        assert err == 0
        assert out[:upto].tobytes() == raw[:upto]
        if value_mode is not None:
            assert (st["value_steps"] > 0) == value_mode, st
    return st


def page_of(table, column):
    """The only data page of `column` in a one-row-group, V1, Snappy Parquet file of `table`: (compressed stream, decoded bytes)."""
    from horaedb_b200 import _ffi
    sink = io.BytesIO()
    pq.write_table(table, sink, compression="snappy", data_page_version="1.0", use_dictionary=False, row_group_size=len(table))
    data = sink.getvalue()
    ci = table.schema.names.index(column)
    ch = _ffi.parquet_chunk_info(data, 0, ci)
    assert ch["num_pages"] == 1 and ch["codec"] == 1
    comp = data[ch["first_page_payload_offset"]:ch["data_page_offset"] + ch["total_compressed_size"]]
    return comp, pa.Codec("snappy").decompress(comp, decompressed_size=_ulen(comp), asbytes=True)


def _ulen(b):
    v, sh, i = 0, 0, 0
    while True:
        v |= (b[i] & 0x7F) << sh
        if not b[i] & 0x80:
            return v
        i, sh = i + 1, sh + 7


def bench_ts_page():
    from horaedb_b200 import sstgen
    sid, ts, value, tag = sstgen.synth_columns(0, 9, 1000, 1000, sstgen.SEED)
    t = pa.table([pa.array(sid[:8192]), pa.array(ts[:8192])], schema=pa.schema([sstgen.METRIC_SCHEMA.field("series_id"),
                                                                               sstgen.METRIC_SCHEMA.field("ts")]))
    return page_of(t, "ts")


def test_bench_ts_page_level_prefix_and_full_decode(emu):
    comp, raw = bench_ts_page()
    # a nullable column's V1 page starts with its definition levels: a 4-byte length and one RLE run (a 3-byte header for 8 192 rows
    # and the level byte), so on the benchmark's pages the values start at byte 8; other phases are covered below
    prefix = 4 + int.from_bytes(raw[:4], "little")
    assert (len(raw) - prefix) == 8192 * 8 and prefix == 8
    st = check(emu, comp, raw, value_mode=True)
    assert st["value_steps"] * 2 > st["steps"]                    # most of the page goes through value mode
    _, _, off = run(emu, comp, len(raw), vmode=False)
    assert st["steps"] < off["steps"] * 0.8


@pytest.mark.parametrize("stop_at", [base + d for base in (8, 12_008) for d in (1, 100, 255, 256, 257)])
def test_bench_ts_page_partial(emu, stop_at):
    """stop_at inside a value-mode batch and on a batch's last byte: the prefix the consumer reads is exact."""
    comp, raw = bench_ts_page()
    check(emu, comp, raw, value_mode=True if stop_at > 12_000 else None, stop_at=stop_at)


@pytest.mark.parametrize("phase", range(8))
def test_value_start_phase(emu, phase):
    s = Stream(phase).rand(phase + 8).pairs(600, L=(1, 2), back=(1, 3, 40))
    check(emu, s.bytes(), bytes(s.out), value_mode=True)


@pytest.mark.parametrize("L", [1, 2, 3, 4, 7])
def test_literal_length(emu, L):
    """Literals of 1-4 bytes pair with a copy of 8 - L >= 4 bytes (Snappy's shortest copy); a 7-byte literal needs a 1-byte copy, which
    value mode leaves to word mode."""
    s = Stream(L).rand(8).pairs(500, L=L, back=(1, 2))
    check(emu, s.bytes(), bytes(s.out), value_mode=L <= 4)


@pytest.mark.parametrize("back", [1, 2, 1000, 8000])
def test_copy_offsets(emu, back):
    """Offsets of 8 and 16 bytes (sources inside the batch), 8 000 (the page's output in global memory) and 64 000 (beyond the ring)."""
    s = Stream(back).rand(8 * back + 5).pairs(700, L=(1, 2), back=back)
    check(emu, s.bytes(), bytes(s.out), value_mode=True)


def test_mixed_sources_and_literal_lengths(emu):
    s = Stream(3).rand(65_000).pairs(2000, L=(1, 2, 3, 4), back=(1, 2, 5, 31, 32, 33, 255, 256, 1000, 8000))
    check(emu, s.bytes(), bytes(s.out), value_mode=True)


def test_parent_chain_of_32(emu):
    """Every value copies the one before it: one chain through all 32 lanes of a batch, with literal bytes of 1-4 along it."""
    s = Stream(4).rand(8)
    for i in range(400):
        s.pair(1 + (i * 7) % 4, 1)
    check(emu, s.bytes(), bytes(s.out), value_mode=True)


@pytest.mark.parametrize("shape", ["span_two_values", "copy5", "copy12"])
def test_pairs_that_fall_back_mid_batch(emu, shape):
    s = Stream(5).rand(16)
    for r in range(12):
        s.pairs(45, L=(1, 2), back=(1, 2))
        if shape == "span_two_values":
            s.rand(1).copy(8, 15)                                  # bytes 1..7 of one value and all of the next
        elif shape == "copy5":
            s.rand(3).copy(16, 5).rand(1).copy(8, 7)               # 3 + 5 = 8 but 5-byte copy at a phase value mode does not expect
        else:
            s.rand(1).copy(16, 12).rand(3)                         # 1 + 12 + 3 = 16: two values, realigned
    s.pairs(45)
    st = check(emu, s.bytes(), bytes(s.out), value_mode=True)
    assert st["value_steps"] >= 12                                 # value mode resumes after every break


def test_long_literal_between_value_runs(emu):
    s = Stream(6).rand(8).pairs(300).rand(100).pairs(300, L=(1, 2)).rand(61).pairs(300, back=(1, 4))
    check(emu, s.bytes(), bytes(s.out), value_mode=True)


def test_nullable_column_with_nulls(emu):
    rng = np.random.default_rng(8)
    v = (1_700_000_000_000 + np.arange(8192) * 1000 + rng.integers(0, 300, 8192)).astype(np.int64)
    mask = rng.random(8192) < 0.05
    t = pa.table({"v": pa.array(v, mask=mask)})
    comp, raw = page_of(t, "v")
    check(emu, comp, raw, value_mode=True)


@pytest.mark.parametrize("phase", [0, 3])
def test_ring_wrap_and_window_edges(emu, phase):
    """Many ring wraps (4 KiB of output each 16 batches) and windows that end inside a pair (literal in, copy out)."""
    s = Stream(9 + phase).rand(8 + phase)
    for i in range(3000):
        s.pair(1 + (i % 3 == 0), 1 + (i % 7 == 0) * 300)
        if i % 97 == 0:
            s.rand(5).copy(8, 3)                                   # shift the pair grid against the window by 8 bytes
    check(emu, s.bytes(), bytes(s.out), value_mode=True)


def _errors(lib, comp, ulen):
    return {run(lib, comp, ulen, order=o, vmode=v)[0] for o in ORDERS for v in (False, True)}


@pytest.mark.parametrize("cut", [0.3, 0.5, 0.77, 0.999])
def test_truncated_stream_same_error(emu, cut):
    s = Stream(10).rand(8).pairs(800, L=(1, 2), back=(1, 1000))
    comp = s.bytes()
    errs = _errors(emu, comp[: int(len(comp) * cut)], len(s.out))
    assert len(errs) == 1 and errs != {0}


@pytest.mark.parametrize("bad", ["offset0", "past_start"])
def test_bad_offset_same_error(emu, bad):
    s = Stream(11).rand(8).pairs(100)
    k = len(s.out)
    s.rand(1)
    s.copy(0 if bad == "offset0" else 8 * (k // 8 + 2), 7, check=False)
    s.out += bytes(7)                                              # the page's declared length counts the copy
    comp = s.bytes()
    errs = _errors(emu, comp, len(s.out))
    assert errs == {103}


@pytest.mark.parametrize("seed", range(6))
def test_damaged_streams_decode_as_without_value_mode(emu, seed):
    """Bytes overwritten, bits flipped and tails cut in value-pair streams: value mode on and off give the same error code and, when the
    decode succeeds, the same bytes."""
    rng = np.random.default_rng(100 + seed)
    s = Stream(seed).rand(8).pairs(900, L=(1, 2, 3), back=(1, 2, 100, 1000))
    clean = s.bytes()
    for trial in range(12):
        bad = bytearray(clean)
        kind = trial % 3
        if kind == 0:
            for p in rng.integers(3, len(bad), 3):
                bad[p] = int(rng.integers(0, 256))
        elif kind == 1:
            for p in rng.integers(3, len(bad), 4):
                bad[p] ^= 1 << int(rng.integers(0, 8))
        else:
            bad = bad[: int(rng.integers(3, len(bad)))]
        ref_err, ref_out, _ = run(emu, bytes(bad), len(s.out), vmode=False)
        for order in ORDERS:
            err, out, _ = run(emu, bytes(bad), len(s.out), order=order)
            assert err == ref_err, (trial, order)
            if err == 0:
                assert out[: len(s.out)].tobytes() == ref_out[: len(s.out)].tobytes()


def _periodic_page():
    """160 KB of random values repeating every 65 600 bytes: a whole-page match finder copies across every 64 KiB boundary with offsets
    above 65 535"""
    rng = np.random.default_rng(12)
    return np.resize(rng.random(8200), 20_000).tobytes()


FOREIGN = dict(fs.SNAPPY_ENCODERS, lopsided=lambda raw, seed=0: fs.snappy_lopsided(raw, len(raw) * 3 // 5),
               literals_anywhere=lambda raw, seed=0: fs.snappy_literals_split(raw, [1, 2, len(raw) // 3, len(raw) - 1], hdr=4))


@pytest.mark.parametrize("page", ["bench_ts", "periodic"])
@pytest.mark.parametrize("name", sorted(FOREIGN))
def test_streams_of_other_encoders(emu, name, page):
    """The encoders of tests/foreign_streams.py on the benchmark's timestamp page and on a page over 64 KiB with far matches: the
    decoder gives the page's bytes in both lane orders, value mode on or off, and the stream holds what the encoder claims"""
    raw = bench_ts_page()[1] if page == "bench_ts" else _periodic_page()
    comp, counts = FOREIGN[name](raw)
    assert pa.Codec("snappy").decompress(comp, decompressed_size=len(raw), asbytes=True) == raw
    check(emu, comp, raw, value_mode=None)
    _, out, _ = run(emu, comp, len(raw), vmode=False)
    assert out[:len(raw)].tobytes() == raw
    if page == "periodic" and name in ("one_window", "copy4_everywhere"):
        assert counts["offset_over_64k"] > 0 and counts["copy_across_64k"] > 0, counts
    if name in ("short_copies", "random_parse"):
        assert counts["copy_under_4"] > 0
    if name == "wide_literal_headers":
        assert counts["wide_literal_header"] > 0
