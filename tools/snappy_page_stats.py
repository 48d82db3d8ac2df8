"""Per-page counters of the Snappy decoder on the benchmark's own SST pages, without a GPU.

Writes one SST the way bench.py does (config 2: 6 250 series x 1 000 points, Snappy, 8 192-row row groups), takes the data page of
each of its four metric columns in the first N row groups, and runs it through the product decoder (horaedb_b200/csrc/snappy_core.h)
compiled for the CPU by tests/emu/snappy_value_emu.cpp.  Prints, per column and per page: windows staged, steps (warp batches), value-mode
steps, elements and output bytes.  Value mode is on for the 8-byte columns, as in snappy_pages_kernel; --no-value-mode turns it off
everywhere, which is the decoder without it.

    python tools/snappy_page_stats.py [--row-groups 24] [--no-value-mode]
"""
import argparse
import ctypes as C
import io
import os
import subprocess
import sys
import tempfile

import numpy as np
import pyarrow.parquet as pq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from horaedb_b200 import _ffi, sstgen  # noqa: E402

COLUMNS = ("series_id", "ts", "value", "tag")
EIGHT_BYTE = (2, 5)          # Parquet INT64, DOUBLE
FIELDS = ("windows", "steps", "elements", "word_steps", "bytes", "parent_searches", "stage_hits", "value_steps")


def build_emu(tmp):
    out = os.path.join(tmp, "libsnappy_emu.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wno-unknown-pragmas", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "emu", "snappy_value_emu.cpp")])
    lib = C.CDLL(out)
    lib.emu_snappy_page.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_long)]
    lib.emu_snappy_page.restype = C.c_int
    lib.emu_set_value_mode.argtypes = [C.c_int]
    return lib


def varint(b):
    v, sh, i = 0, 0, 0
    while True:
        v |= (b[i] & 0x7F) << sh
        if not b[i] & 0x80:
            return v
        i, sh = i + 1, sh + 7


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--row-groups", type=int, default=24)
    ap.add_argument("--no-value-mode", action="store_true")
    args = ap.parse_args()
    data, _ = sstgen.synth_sst(0, 6250, 1000, 1000, seq=1_000_000)      # bench.py's first file
    names = pq.ParquetFile(io.BytesIO(data)).schema_arrow.names
    summary = _ffi.parquet_inspect(data)
    nrg = min(args.row_groups, summary["num_row_groups"])
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_emu(tmp)
        print(f"{'column':10} {'pages':>5} {'comp B':>8} {'out B':>8} {'windows':>8} {'steps':>7} {'value':>7} {'word':>7} {'elements':>9} {'B/step':>7}")
        for ci, name in enumerate(COLUMNS):
            col = names.index(name)
            tot = np.zeros(len(FIELDS), dtype=np.int64)
            comp_b = out_b = pages = 0
            for rg in range(nrg):
                ch = _ffi.parquet_chunk_info(data, rg, col)
                if ch["num_pages"] != 1 or ch["codec"] != 1:
                    continue
                page = data[ch["first_page_payload_offset"]:ch["data_page_offset"] + ch["total_compressed_size"]]
                ulen = varint(page)
                lib.emu_set_value_mode(0 if args.no_value_mode else int(ch["physical_type"] in EIGHT_BYTE))
                out = np.zeros(ulen + 320, np.uint8)
                n = C.c_long(0)
                err = lib.emu_snappy_page(page, len(page), out.ctypes.data, ulen, 0xFFFFFFFF, C.byref(n))
                if err:
                    raise SystemExit(f"{name} row group {rg}: decoder error {err}")
                st = (C.c_long * len(FIELDS))()
                lib.emu_stats(st)
                tot += np.array(st[:], dtype=np.int64)
                comp_b += len(page)
                out_b += ulen
                pages += 1
            f = dict(zip(FIELDS, tot / max(pages, 1)))
            print(f"{name:10} {pages:5d} {comp_b / max(pages, 1):8.0f} {out_b / max(pages, 1):8.0f} {f['windows']:8.1f} {f['steps']:7.1f} "
                  f"{f['value_steps']:7.1f} {f['word_steps']:7.1f} {f['elements']:9.1f} {f['bytes'] / max(f['steps'], 1):7.1f}")


if __name__ == "__main__":
    main()
