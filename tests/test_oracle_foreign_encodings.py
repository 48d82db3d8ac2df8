"""The C oracle's page decoders (oracle/horae_oracle.c) on the re-laid-out files of tests/test_gpu_foreign_encodings.py: every file
decodes like the oracle reads the source, and like pyarrow reads it wherever pyarrow accepts the layout.  Building the files runs
tests/page_encodings.py's self-checks (the baseline layout gives back the source byte for byte, pyarrow reads the result equal to the
source), and the layouts' counts show that each feature a layout claims occurs in the files the GPU tests read."""
import io

import pyarrow.parquet as pq
import pytest

import page_encodings as pe
from helpers import arrays_equal
from test_gpu_foreign_encodings import (LAYOUTS, METRIC, PYARROW_REFUSES, all_types_schema, all_types_src, binary_src, bit_packed_levels, fused_source,
                                        metric_src, overlapping_sources, recoded, required_src)
from oracle import oracle


def _sources():
    return [(s, METRIC.arrow_schema) for s in overlapping_sources() + [fused_source()]] + \
        [(all_types_src(v2), all_types_schema().arrow_schema) for v2 in (False, True)]


def _same_as_source(data, src, schema, pyarrow_reads=True):
    got = oracle.decode_sst(data, schema)
    exp = oracle.decode_sst(src, schema)
    ref = pq.read_table(io.BytesIO(src))
    assert got.num_rows == exp.num_rows == ref.num_rows
    for c in schema.names:
        assert arrays_equal(got[c], exp[c]) and arrays_equal(got[c], ref[c]), c
    if pyarrow_reads:
        back = pq.read_table(io.BytesIO(data))
        for c in schema.names:
            assert arrays_equal(back[c], ref[c]), c


@pytest.mark.parametrize("stats", [False, True])
@pytest.mark.parametrize("name", list(LAYOUTS))
def test_oracle_reads_recoded_files(name, stats):
    for src, schema in _sources():
        _same_as_source(recoded(src, name, stats)[0], src, schema, name not in PYARROW_REFUSES)


def test_pyarrow_refuses_the_listed_layouts():
    """INT32 deltas in 64-bit arithmetic (widths of 33 bits): pyarrow 24 cannot read the full-range INT32 columns; the oracle and the
    engine take the deltas modulo 2^32 as the spec's wrapping arithmetic allows.  Every other layout pyarrow reads."""
    for name in PYARROW_REFUSES:
        with pytest.raises(OSError):
            pq.read_table(io.BytesIO(recoded(all_types_src(False), name)[0]))


# the features each layout must show on the files above (summed over their chunks)
_RUNS = ["run_end_mod8_%d" % i for i in range(8)]
FEATURES = {
    "delta_128_1": ["delta_128_1", "count_0", "count_1", "count_block", "count_block_plus_1", "varint_10_bytes"],
    "delta_256_8": ["delta_256_8", "count_block", "count_block_plus_1"], "delta_256_2": ["delta_256_2", "count_block_plus_1"],
    "delta_1024_8": ["delta_1024_8", "count_block", "count_block_plus_1"], "delta_2048_16": ["delta_2048_16", "count_1"],
    "delta_4096_64": ["delta_4096_64", "count_1"], "delta_wide": ["width_64"], "delta_junk": ["junk_unused_width", "ones_in_padding"],
    "delta_i32_64bit": ["int32_width_over_32", "min_delta_outside_i32"],
    "dict_rle": ["rle_run_of_1", "width_0_one_entry"] + _RUNS, "dict_packed": ["packed_groups_1", "packed_groups_63", "packed_uniform"],
    "dict_alternate": ["rle_run", "packed_run", "packed_uniform"] + _RUNS, "dict_mod8": ["rle_run_of_1", "packed_run"] + _RUNS,
    "dict_wide": ["index_width_32"], "dict_wide_23": ["index_width_23"], "dict_plain_dictionary": ["plain_dictionary_ids"],
    "dict_fallback": ["fallback_to_plain"], "dict_unnamed": ["dictionary_page_unnamed"], "dict_pad_ones": ["nonzero_padding"],
    "levels_rle": ["all_valid_chunk", "rle_run_of_1"], "levels_short_rle": ["all_valid_chunk", "rle_run_of_1"] + _RUNS,
    "levels_packed": ["all_valid_chunk", "packed_groups_1", "packed_uniform"], "levels_alternate": ["rle_run", "packed_uniform"] + _RUNS,
    "levels_mod8": ["rle_run_of_1", "packed_run"] + _RUNS, "pages_1_7": ["pages_of_1_and_7"],
    "mixed": ["mixed_chunk", "delta_256_8", "rle_run", "packed_run"],
}


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_layouts_emit_their_features(name):
    assert set(FEATURES) == set(LAYOUTS)
    counts = {}
    for src, _ in _sources():
        for k, v in recoded(src, name)[1].items():
            counts[k] = counts.get(k, 0) + v
    for f in FEATURES[name]:
        assert counts.get(f, 0) > 0, (f, sorted(counts))


@pytest.mark.parametrize("name", [n for n in LAYOUTS if n.startswith(("delta_", "dict_"))])
def test_binary_layouts_emit_their_features(name):
    """on the Binary source (the oracle does not read Binary columns; building the files checks them against pyarrow): the DELTA layouts
    write DELTA_LENGTH_BYTE_ARRAY and DELTA_BYTE_ARRAY pages with shared prefixes in their geometry, the dictionary layouts Binary
    dictionaries"""
    counts = {}
    for v2 in (False, True):
        for k, v in recoded(binary_src(v2), name)[1].items():
            counts[k] = counts.get(k, 0) + v
    want = ["binary_dictionary"] if name.startswith("dict_") else ["dlba_page", "dba_page", "dba_shared_prefix"]
    want += {"delta_junk": ["junk_unused_width", "ones_in_padding"], "dict_pad_ones": ["nonzero_padding"],
             "delta_4096_64": ["delta_4096_64"], "delta_128_1": ["delta_128_1", "count_block_plus_1"]}.get(name, [])
    for f in want:
        assert counts.get(f, 0) > 0, (f, sorted(counts))


def test_short_rle_levels_are_longer_than_a_bit_per_row():
    """levels_short_rle writes all-valid levels at about 2 bytes per row: far past the `rows + 16` bytes a gate once assumed"""
    data = recoded(fused_source(), "levels_short_rle")[0]
    for ch in pe.chunks_of(fused_source())[0][:1]:
        n = len(ch.levels)
        assert len(pe.hybrid_encode(ch.levels, 1, "short_rle")) > n + 16
    assert len(data) > len(fused_source())


def test_oracle_refuses_bit_packed_levels_and_reads_a_bit_packed_label():
    src = metric_src(0, 4, 100, 61, nulls=0.1)
    data = pe.recode(src, lambda c: bit_packed_levels(c, {}), pyarrow_reads=False)
    with pytest.raises(Exception, match="definition level encoding 4"):
        oracle.decode_sst(data, METRIC.arrow_schema)
    req = required_src()
    got = oracle.decode_sst(pe.recode(req, lambda c: bit_packed_levels(c, {})), METRIC.arrow_schema)
    ref = pq.read_table(io.BytesIO(req))
    for c in ("series_id", "ts", "value", "tag"):
        assert arrays_equal(got[c], ref[c]), c
