"""TEST INFRASTRUCTURE: damaged SSTs whose Binary columns are dictionary-encoded or DELTA_BYTE_ARRAY, through the emulated library with
guard pages behind every device allocation (the harness and the damage model of fuzz_engine.py).  Damage lands in dictionary pages, index
runs, both DELTA_BYTE_ARRAY length runs, suffix bytes, page headers and the footer.  Every call (scan with and without a predicate, a
single-file scan, hg_compact_open) must end in a result or an HgError; a kernel that reads or writes outside its buffers is a crash here,
reported with kernel, block and thread.

    python tests/emu/fuzz_binary_encodings.py SEED ITERATIONS [KIND ...]      KIND: dict dict-append dba dba-append

dict: PLAIN dictionary page + RLE_DICTIONARY indices (enable_dict); dba: DELTA_BYTE_ARRAY; -append: UpdateMode::Append (BytesMergeOperator)."""
import ctypes as C
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import fuzz_engine  # noqa: E402  (builds the emulated library and points horaedb_b200._ffi at it)
import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402

from horaedb_b200 import _ffi, sstgen  # noqa: E402
from horaedb_b200._ffi import Engine, HgError, SchemaHandle, SstInput  # noqa: E402
from horaedb_b200.config import ColumnOptions, ParquetEncoding, WriteConfig  # noqa: E402
from horaedb_b200.types import StorageSchema, UpdateMode  # noqa: E402


def make_case(kind, rng):
    """-> (schema handle, [SST bytes, one per codec])"""
    mode = UpdateMode.Append if kind.endswith("-append") else UpdateMode.Overwrite
    user = pa.schema([pa.field("pk1", pa.uint64()), pa.field("pk2", pa.int32()), pa.field("blob", pa.binary()), pa.field("idx", pa.binary())])
    sch = StorageSchema.try_new(user, 2, mode)
    files = []
    for i, codec in enumerate(("none", "snappy", "zstd")):
        pk1 = np.unique(rng.integers(0, 4000, 1200))
        cols = [pa.array(pk1.astype(np.uint64)), pa.array((pk1 % 5 - 2).astype(np.int32)),
                pa.array([None if (int(k) + i) % 7 == 0 else b"host-%04d/" % (int(k) // 9) + rng.bytes(int(rng.integers(0, 12))) for k in pk1], pa.binary()),
                pa.array([b"label-%d" % int(rng.integers(0, 5)) for _ in pk1], pa.binary())]
        if kind.startswith("dict"):
            cfg = WriteConfig(compression=codec, max_row_group_size=500, enable_dict=True)
        elif kind.startswith("dba"):
            cfg = WriteConfig(compression=codec, max_row_group_size=500,
                              column_options={c: ColumnOptions(encoding=ParquetEncoding.DeltaByteArray) for c in ("blob", "idx")})
        else:
            raise SystemExit("unknown kind " + kind)
        files.append(sstgen.write_sst(sch, pa.RecordBatch.from_arrays(cols, schema=user), 50 + i, cfg, presorted=True))
    return SchemaHandle(sch.arrow_schema, 2, mode), files


def main():
    seed, iters = int(sys.argv[1]), int(sys.argv[2])
    kinds = sys.argv[3:] or ["dict", "dict-append", "dba", "dba-append"]
    rng = np.random.default_rng(seed)
    eng = Engine(device=0)
    lib = _ffi.lib()
    tmp = tempfile.mkdtemp(prefix="horae_fuzz_bin_")
    accepted = rejected = 0
    for kind in kinds:
        handle, files = make_case(kind, rng)
        for it in range(iters):
            which = it % len(files)
            bad = fuzz_engine.damage(rng, files[which])
            with open(os.path.join(tmp, "current.sst"), "wb") as f:          # the input of a crash stays on disk
                f.write(bad)
            ins = [SstInput(id=10_000 + it, data=bad), SstInput(id=5, data=files[(which + 1) % len(files)])]
            op = it % 4
            try:
                if op == 0:
                    eng.scan(handle, ins).read_all()
                elif op == 1:
                    eng.scan(handle, ins, [("pk2", "ge", 0)]).read_all()
                elif op == 2:
                    eng.scan(handle, ins[:1], [], None, True).read_all()
                else:
                    eng.compact(handle, ins).read_all()
                accepted += 1
            except HgError:
                rejected += 1
            line = C.c_int()
            sched = lib.emu_take_error(C.byref(line))            # threads that left a block through different barriers
            if sched:
                raise SystemExit(f"{kind} file {it} (op {op}): emulated scheduler error {sched} at source line {line.value}")
        print(f"{kind}: done ({iters} files)", flush=True)
    print(f"accepted {accepted} rejected {rejected}")


if __name__ == "__main__":
    main()
