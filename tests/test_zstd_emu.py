"""The product's warp-level Zstandard decoder (horaedb_b200/csrc/zstd_core.h — the text nvcc compiles for sm_90a) executed on the
CPU (tests/emu/zstd_emu.cpp: 32 coroutines, warp collectives as rendezvous).  Streams come from libzstd through pyarrow — the
compressor behind pyarrow's Parquet ZSTD pages and (as zstd 0.13.2) behind parquet-rs in the reference (config.rs:78-94).  Levels 1, 3
and 9 change which features a frame uses: raw / RLE / Huffman literals (1 and 4 streams, direct and FSE-compressed weights), predefined /
RLE / FSE-compressed / repeated sequence tables, repeat offsets, overlapping matches, several blocks per frame."""
import ctypes as C
import os
import subprocess

import numpy as np
import pyarrow as pa
import pytest

import foreign_streams as fs

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "zstd_emu.cpp")
DEPS = [SRC, os.path.join(HERE, "emu", "warp_emu.h"), os.path.join(HERE, "..", "horaedb_b200", "csrc", "zstd_core.h")]
OUT = os.path.join(HERE, "emu", "_build", "libzstd_emu.so")
GUARD = 0xEE


@pytest.fixture(scope="module")
def emu():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", OUT, SRC])
    lib = C.CDLL(OUT)
    lib.emu_zstd_page.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_long)]
    lib.emu_zstd_page.restype = C.c_int
    return lib


def decode(lib, comp, ulen):
    out = np.full(ulen + 256, GUARD, dtype=np.uint8)
    n = C.c_long(0)
    err = lib.emu_zstd_page(comp, len(comp), out.ctypes.data, ulen, C.byref(n))
    return err, out


def _cases():
    rng = np.random.default_rng(5)
    n = 8192
    prefix = b"\x02\x00\x00\x00\x03\x10"
    ts = (1_700_000_000_000 + np.tile(np.arange(1000), 9)[:n].astype(np.int64) * 1000 + rng.integers(0, 500, n)).astype(np.int64)
    return {
        "empty": b"", "three_bytes": b"abc", "short_run": b"a" * 70,
        "jitter_ts": prefix + ts.tobytes(),
        "series_id": prefix + np.repeat(np.arange(9, dtype=np.uint64) + 77, 1000)[:n].tobytes(),
        "tag_u32": prefix + (np.repeat(np.arange(9), 1000)[:n] % 16).astype(np.uint32).tobytes(),
        "random": rng.integers(0, 2**63, n, dtype=np.uint64).tobytes(),               # raw block
        "sawtooth": ((np.arange(n, dtype=np.uint64) % 1000) * 37).tobytes(),
        "slow_counter": (np.arange(n, dtype=np.uint64) // 3).tobytes(),
        "few_values": rng.choice(rng.integers(0, 2**60, 5, dtype=np.uint64), n).tobytes(),
        "small_u32": rng.integers(0, 16, n).astype(np.uint32).tobytes(),
        "text": (b"the quick brown fox jumps over the lazy dog. " * 500)[:20000],
        "f64_round": np.round(rng.random(n), 2).tobytes(),
        "skewed_bytes_300k": rng.integers(0, 50, 300_000).astype(np.uint8).tobytes(),   # three blocks, Huffman literals in four streams
    }


CASES = _cases()


@pytest.mark.parametrize("level", [1, 3, 9])
@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_zstd_decoder_matches_input(emu, name, level):
    raw = CASES[name]
    comp = pa.Codec("zstd", compression_level=level).compress(raw, asbytes=True)
    err, out = decode(emu, comp, len(raw))
    assert err == 0
    assert bytes(out[:len(raw)]) == raw
    assert (out[len(raw):] == GUARD).all()


def test_emulated_zstd_decoder_rejects_malformed(emu):
    raw = CASES["jitter_ts"]
    comp = pa.Codec("zstd").compress(raw, asbytes=True)
    err, _ = decode(emu, comp, len(raw) + 1)                   # the page header promises another size
    assert err != 0
    err, _ = decode(emu, comp[: len(comp) // 2], len(raw))     # truncated frame
    assert err != 0
    bad = bytearray(comp)
    bad[0] ^= 0xFF                                             # magic
    err, _ = decode(emu, bytes(bad), len(raw))
    assert err == 202


@pytest.mark.parametrize("enc", sorted(fs.ZSTD_ENCODERS))
@pytest.mark.parametrize("name", ["empty", "jitter_ts", "random", "tag_u32", "skewed_bytes_300k"])
def test_emulated_zstd_decoder_on_other_frame_shapes(emu, name, enc):
    """Streaming frames (no content size, flushed into many small blocks), levels -7 to 22, several frames per page, skippable frames,
    the checksum flag, raw / RLE blocks only (tests/foreign_streams.py): libzstd and the decoder agree"""
    raw = CASES[name]
    comp = fs.ZSTD_ENCODERS[enc](raw)
    if raw:
        assert pa.Codec("zstd").decompress(comp, decompressed_size=len(raw), asbytes=True) == raw
    err, out = decode(emu, comp, len(raw))
    assert err == 0
    assert bytes(out[:len(raw)]) == raw
    assert (out[len(raw):] == GUARD).all()
