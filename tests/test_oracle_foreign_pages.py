"""The C oracle's Snappy and Zstandard readers (oracle/horae_oracle.c, oracle/zstd_oracle.h) on the recoded files of
tests/test_gpu_foreign_pages.py: every file decodes like pyarrow reads it and like the oracle reads the source.  Building the files runs
tests/page_recode.py's self-checks on each (identity round trip, pyarrow equality, every stream vouched for by libsnappy / libzstd), and
the encoders' counts show that each feature a case claims occurs in the files the GPU tests read."""
import io

import pyarrow.parquet as pq
import pytest

import foreign_streams as fs
from helpers import arrays_equal
from test_gpu_foreign_pages import (ENCODERS, METRIC, SNAPPY_NAMES, _overlapping_sources, _stored_file, all_types_schema,
                                    all_types_src, fused_sources, recoded)
from oracle import oracle


def _same_as_source(data, src, schema):
    got = oracle.decode_sst(data, schema)
    exp = oracle.decode_sst(src, schema)
    ref = pq.read_table(io.BytesIO(data))
    assert got.num_rows == exp.num_rows == ref.num_rows
    for c in schema.names:
        assert arrays_equal(got[c], exp[c]) and arrays_equal(got[c], ref[c]), c


@pytest.mark.parametrize("name", list(ENCODERS))
def test_oracle_reads_recoded_files(name):
    for src in _overlapping_sources():
        _same_as_source(recoded(src, name)[0], src, METRIC.arrow_schema)
    _same_as_source(recoded(all_types_src(), name)[0], all_types_src(), all_types_schema().arrow_schema)
    for src in fused_sources():
        _same_as_source(recoded(src, name)[0], src, METRIC.arrow_schema)


# the features each encoder must show on the files above (summed over their pages)
FEATURES = {
    "copy1_only": ["copy1"], "copy2_only": ["copy2", "copy2_where_copy1_fits"], "copy4_everywhere": ["copy4", "offset_over_64k"],
    "one_window": ["copy_across_64k", "offset_over_64k"], "short_copies": ["copy_under_4", "copy_across_64k"],
    "wide_literal_headers": ["wide_literal_header"], "random_parse": ["copy_under_4", "copy_across_64k"],
    "lopsided": ["copy_across_64k"], "literals_anywhere": ["literal_across_64k"],
}


@pytest.mark.parametrize("name", SNAPPY_NAMES)
def test_snappy_encoders_emit_their_features(name):
    counts = {}
    for src in fused_sources() + [all_types_src()] + _overlapping_sources():
        for k, v in recoded(src, name)[1].items():
            counts[k] = counts.get(k, 0) + v
    for f in FEATURES[name]:
        assert counts.get(f, 0) > 0, (f, counts)


def test_zstd_frame_shapes():
    """what each Zstandard encoder writes into a page of the files: streaming frames start 0x00 (a window descriptor, no content size),
    one-shot ones are Single_Segment (0x20 set), several frames per page, skippable frames around the data, the checksum flag"""
    from page_recode import page_streams
    page = page_streams(_overlapping_sources()[0], 1)[0][0]
    assert len(page) > 1024
    single = lambda n: lambda g: len(g) == n and all(x & 0x20 and not x & 0x04 for x in g)
    expect = {"stream": lambda g: g == [0x00], "stream_flush_1k": lambda g: g == [0x00], "stream_flush_7k": lambda g: g == [0x00],
              "two_frames": single(2), "three_frames": single(3), "checksum": lambda g: len(g) == 1 and g[0] & 0x24 == 0x24,
              "skippable_around": lambda g: g[0] == g[2] == "skip" and len(g) == 3 and g[1] & 0x20, "raw_rle": single(1),
              "raw_rle_window": lambda g: g == [0x00]}
    for lv in (-7, -1, 1, 3, 9, 19, 22):
        expect[f"level_{lv}"] = single(1)
    assert set(expect) == set(fs.ZSTD_ENCODERS)
    for name, ok in expect.items():
        got = fs.zstd_frame_header_bytes(fs.ZSTD_ENCODERS[name](page))
        assert ok(got), (name, got)


@pytest.mark.parametrize("case", ["one_literal", "n0=0", "n0=1", "n0=rows/2", "n0=rows-1", "inside_prefix", "prefix_too_short",
                                  "inside_value", "three_literals"])
def test_oracle_reads_stored_splits(case):
    src, data, counts = _stored_file(case)
    assert counts
    _same_as_source(data, src, METRIC.arrow_schema)
