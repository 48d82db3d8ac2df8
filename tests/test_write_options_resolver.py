"""Host only: `config.resolve_column_options` — WriteConfig + the storage schema -> the per-column options of the GPU SST writer — and
which writes of `ObjectBasedStorage` it sends to the GPU writer (an engine stand-in records the calls; refused configurations keep the
host writer)."""
import ctypes as C

import pyarrow as pa
import pyarrow.parquet as pq

from horaedb_b200 import _ffi
from horaedb_b200.config import ColumnOptions, ParquetCompression, ParquetEncoding, StorageConfig, WriteConfig, resolve_column_options
from horaedb_b200.types import StorageSchema

from helpers import arrow_schema, record_batch

D, P = ParquetEncoding.DeltaBinaryPacked, ParquetEncoding.Plain
USER = arrow_schema([("k", "uint64"), ("ts", "int64"), ("v", "float64"), ("t", "uint16")])
SCHEMA = StorageSchema.try_new(USER, 2).arrow_schema          # + __seq__ (u64), __reserved__ (u64)


def test_struct_layouts():
    assert C.sizeof(_ffi.HgColumnWriteOpts) == 4
    assert C.sizeof(_ffi.HgWriteProps) == 24 and _ffi.HgWriteProps.columns.offset == 16


def test_default_config_is_plain_with_the_table_codec():
    assert resolve_column_options(WriteConfig(), SCHEMA) == [(P, False, "snappy")] * 6
    assert resolve_column_options(WriteConfig(compression=ParquetCompression.Zstd), SCHEMA) == [(P, False, "zstd")] * 6


def test_column_options_override_the_table_fields():
    cfg = WriteConfig(encoding=D, enable_dict=True, compression="none",
                      column_options={"v": ColumnOptions(encoding=P, enable_dict=False, compression="zstd"),
                                      "__seq__": ColumnOptions(enable_dict=False), "t": ColumnOptions(compression="snappy"),
                                      "nope": ColumnOptions(encoding="RLE")})      # a name outside the schema changes nothing
    assert resolve_column_options(cfg, SCHEMA) == [(D, True, "none"), (D, True, "none"), (P, False, "zstd"), (D, True, "snappy"),
                                                   (D, False, "none"), (D, True, "none")]


def test_dictionary_with_delta_fallback_reaches_the_gpu():
    cfg = WriteConfig(enable_dict=True, column_options={"ts": ColumnOptions(encoding=D)})
    assert resolve_column_options(cfg, SCHEMA)[1] == (D, True, "snappy")


def test_refused_configurations():
    for cfg in (WriteConfig(encoding=D),                                             # DELTA on the f64 column
                WriteConfig(column_options={"v": ColumnOptions(encoding=D)}),
                WriteConfig(encoding=ParquetEncoding.Rle),
                WriteConfig(column_options={"k": ColumnOptions(encoding=ParquetEncoding.RleDictionary)}),
                WriteConfig(column_options={"ts": ColumnOptions(encoding=ParquetEncoding.DeltaByteArray)}),
                WriteConfig(column_options={"ts": ColumnOptions(encoding=ParquetEncoding.DeltaLengthByteArray)}),
                WriteConfig(column_options={"t": ColumnOptions(compression="gzip")}),
                WriteConfig(compression="lz4")):
        assert resolve_column_options(cfg, SCHEMA) is None, cfg
    binary = StorageSchema.try_new(arrow_schema([("k", "uint64"), ("b", "binary")]), 1).arrow_schema
    assert resolve_column_options(WriteConfig(), binary) is None


class _RecordingEngine:
    def __init__(self):
        self.calls = []

    def write_batch(self, schema, batch, sequence, out_path, max_row_group_size=8192, compression="snappy", enable_sorting_columns=True, columns=None):
        self.calls.append(columns)
        with open(out_path, "wb") as f:
            f.write(b"")
        return _ffi.HgFileMeta(size=0, num_rows=batch.num_rows)


def test_storage_sends_resolved_configurations_to_the_gpu_writer(tmp_path):
    from horaedb_b200.storage import ObjectBasedStorage, WriteRequest
    from horaedb_b200.types import TimeRange
    batch = record_batch(USER, {"k": [2, 1], "ts": [5, 6], "v": [0.5, 1.5], "t": [3, None]})
    cases = [(WriteConfig(), True),
             (WriteConfig(enable_dict=True, column_options={"ts": ColumnOptions(encoding=D)}), True),
             (WriteConfig(column_options={"k": ColumnOptions(encoding=D, compression="zstd")}), True),
             (WriteConfig(encoding=D), False),                                       # DELTA on f64: pyarrow (host) refuses it too
             (WriteConfig(column_options={"t": ColumnOptions(compression="gzip")}), False)]
    for i, (cfg, gpu) in enumerate(cases):
        eng = _RecordingEngine()
        st = ObjectBasedStorage(str(tmp_path / str(i)), 1000, USER, 2, StorageConfig(write=cfg), engine=eng)
        try:
            st.write(WriteRequest(batch, TimeRange(0, 10)))
        except Exception:
            assert not gpu                                                           # the host writer's own refusal, as before
        assert (len(eng.calls) == 1) == gpu, cfg
        if gpu:
            assert eng.calls[0] == resolve_column_options(cfg, st.schema_.arrow_schema)
        elif cfg.column_options and "t" in cfg.column_options:
            files = list((tmp_path / str(i)).rglob("*.sst"))
            assert files and pq.ParquetFile(files[0]).metadata.row_group(0).column(3).compression == "GZIP"
