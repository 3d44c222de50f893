"""The PNG edge inputs (tests/png_edge_inputs.py) on the CPU: every builder's stated counts
against the census of its bytes, every valid stream through Python's zlib and cv2 to the intended
bytes and pixels, every refusal as zlib names it and as cv2 reads it with the stream whole, in
1-byte and in 7-byte IDAT chunks, and the host parse accepting all of them for the device to
judge (tests/test_gpu_png_edges.py runs them on the device)."""
import functools
import zlib

import numpy as np
import pytest

import png_decode_inputs as P
import png_edge_inputs as E
from matterport_maskrcnn_with_tensorflow_serving_b200 import png


@functools.lru_cache(maxsize=None)
def _cases():
    return E.all_cases()


@functools.lru_cache(maxsize=None)
def _census():
    return [E.census(c) for c in _cases()]


# every edge the inputs are built for, each of which some file holds at least once
EDGES = (["dist_one_code", "dist_empty", "literal_only", "lit_all_15", "cl_cross",
          "cl16_first_dist", "cl18_138", "hclen_4", "hclen_19", "hlit_257", "hlit_286", "hdist_1",
          "hdist_30", "len284_31", "len285_258", "dist_1", "dist_32506", "dist_far_end",
          "dist_window", "dist_window_plus_1", "dist_past_window", "dist_same_row",
          "dist_earlier_row", "reach_exact", "reach_past", "stored_len_0", "stored_len_1",
          "stored_len_65535", "stored_after_fixed", "stored_after_dynamic", "dense_tiles",
          "false_candidates", "false_to_end", "hlit_287", "hlit_288", "hdist_31", "hdist_32",
          "cl_incomplete", "cl_empty", "cl16_first", "cl_overrun", "lit_over", "lit_incomplete",
          "dist_incomplete", "dist_over", "fixed_286", "fixed_287", "dist_code_30",
          "dist_code_31", "paeth_ab", "paeth_ac", "paeth_bc", "paeth_all", "adam7_rows_gt256",
          "adam7_one_col", "row_1byte_f1", "row_1byte_f3", "row_1byte_f4",
          "error: invalid code -- missing end-of-block"]
         + [f"lit_len_{l}" for l in range(11, 16)] + [f"dist_len_{l}" for l in range(11, 16)]
         + [f"stored_phase_{k}" for k in range(8)] + [f"cinfo_{k}" for k in range(8)])


@pytest.mark.parametrize("builder", E.BUILDERS, ids=lambda b: b.__name__)
def test_builder_counts(builder):
    for case in builder(np.random.default_rng(0)):
        got = E.census(case)
        for key, want in case.counts.items():
            assert want > 0 and got.get(key, 0) >= want, (case.name, key, got.get(key, 0), want)
    if builder is E.lengths:
        assert got["len_base"] == got["len_top"] == 29


def test_the_census_covers_every_edge():
    total = {}
    for c in _census():
        for k, v in c.items():
            total[k] = total.get(k, 0) + v
    missing = [k for k in EDGES if not total.get(k)]
    assert not missing, missing


def test_valid_streams_inflate_to_the_intended_bytes():
    for case in _cases():
        if case.pixels is None or case.raw is None:
            continue
        z = P.zlib_stream(case.blob)
        assert zlib.decompress(z) == case.raw, case.name
        out, blocks = E.walk(z)
        assert out == case.raw and "error" not in blocks[-1], case.name


def test_cv2_decodes_every_valid_file_to_the_intended_pixels():
    for case in _cases():
        if case.pixels is None:
            continue
        z = P.zlib_stream(case.blob)
        for split in (None, 7) if len(z) < 100000 else (None,):
            got = P.cv2_decode(P.with_zlib_stream(case.blob, z, split))
            assert got is not None and np.array_equal(got, case.pixels), (case.name, split)


def test_refusals_as_zlib_names_them_and_cv2_reads_them():
    refused = [c for c in _cases() if c.pixels is None]
    assert len(refused) == 34
    for case in refused:
        z = P.zlib_stream(case.blob)
        _, blocks = E.walk(z)
        err = blocks[-1].get("error")
        assert err, case.name
        if case.status == E.ST_DIST and err == "invalid distance too far back" and \
                blocks[-1]["tokens"][-1][7] > 256 << (z[0] >> 4):
            pass      # past the window: zlib's one-shot inflate has the bytes in its output
        elif case.name == "empty code-length code":
            # inflate takes an empty code-length code and reads one bit per length, all 0: it
            # fails at the missing end-of-block (here: runs out of data first)
            with pytest.raises(zlib.error, match="incomplete or truncated"):
                zlib.decompress(z)
        else:
            with pytest.raises(zlib.error, match=err.replace("(", r"\(")):
                zlib.decompress(z)
        for split, decodes in zip((None, 1, 7), case.cv2):
            assert (P.cv2_decode(P.with_zlib_stream(case.blob, z, split)) is not None) == \
                decodes, (case.name, split)
        assert not all(case.cv2), case.name      # the device refuses what cv2 may refuse


def test_host_parse_accepts_every_file():
    cases = _cases()
    for case in cases:
        hd = png.parse(case.blob)
        assert hd.window == 256 << (P.zlib_stream(case.blob)[0] >> 4)
    plan = png.DecodePlan([c.blob for c in cases])
    assert plan.B == len(cases)


def test_the_finder_restated_finds_every_dynamic_block():
    """candidates() accepts every true dynamic block start (so the device's CAND count can be
    held to it), and the dense and false-header files overfill 4 slots of some tile."""
    for case in _cases():
        z = P.zlib_stream(case.blob)
        if case.pixels is None or len(z) > 20000:
            continue
        cand = set(E.candidates(z))
        _, blocks = E.walk(z)
        assert {b["bit"] for b in blocks if b["type"] == 2} <= cand, case.name
    dense = next(c for c in _cases() if c.name == "one literal per dynamic block")
    cand = E.candidates(P.zlib_stream(dense.blob))
    per = np.bincount(np.asarray(cand) // E.TILE_BITS)
    assert per.max() >= 10
