"""The PNG encoder's edge inputs (tests/png_encode_edge_inputs.py) on the CPU: every builder's
stated counts against the census of the oracle's blocks; the oracle against cv2.imencode byte for
byte, and its deflate body against zlib fed one filtered row per call as libpng feeds it; every
one-mistake variant of the oracle changing some edge image's bytes (the two argued equivalent
changing none); and every file under png_bound (tests/test_gpu_png_encode_edges.py runs the same
images on the device)."""
import functools
import zlib

import numpy as np
import pytest

import png_encode_edge_inputs as E
import png_oracle as P

cv2 = pytest.importorskip("cv2")


@functools.lru_cache(maxsize=None)
def _cases():
    return E.all_cases()


@functools.lru_cache(maxsize=None)
def _encoded():
    return [P.encode(c.img) for c in _cases()]


# every edge the inputs are built for; each is held by some image
EDGES = (["lit_overflow_2", "lit_overflow_4", "lit_overflow_6", "lit_overflow_8",
          "lit_overflow_first", "lit_overflow_middle", "lit_overflow_final", "lit_overflow_full",
          "bl_overflow_2", "bl_overflow_4", "bl_overflow_6", "depth_tie", "full_tie",
          "dist_empty", "dist_one", "eob_only", "one_literal_eob", "stored_tie", "stored_tie_m1",
          "stored_tie_p1", "static_tie", "static_tie_m1", "static_tie_p1", "stretch_at_tile",
          "stretch_at_tile_m1", "stretch_at_tile_p1", "stretch_ends_at_tile", "stretch_3_tiles",
          "sym16383_match_tile_first", "sym16383_match_tile_last", "match_first_in_block",
          "match_last_in_block", "stored_stored", "stored_final", "one_chunk", "adler_n_0",
          "adler_n_m1", "adler_n_p1", "adler_255_tiles"]
         + [f"stretch_258m_r{r}" for r in range(4)] + [f"stored_phase_{k}" for k in range(8)]
         + [f"zlen_mod_{r}" for r in (0, 1, 2, 3, 4, 8191)])


@pytest.mark.parametrize("builder", E.BUILDERS, ids=lambda b: b.__name__)
def test_builder_counts(builder):
    for case in builder(np.random.default_rng(0)):
        got = E.census(P.encode(case.img)[1])
        for key, want in case.counts.items():
            assert want > 0 and got.get(key, 0) >= want, (case.name, key, got.get(key, 0), want)


def test_the_census_covers_every_edge():
    total = {}
    for _, e in _encoded():
        for k, v in E.census(e).items():
            total[k] = max(total.get(k, 0), v) if k == "hdr_bits_max" else total.get(k, 0) + v
    missing = [k for k in EDGES if not total.get(k)]
    assert not missing, missing
    # unreachable, as the builders' docstrings argue
    assert not any(total.get(k) for k in ("lit_overflow_1", "lit_overflow_3", "lit_overflow_5",
                                          "bl_overflow_1", "bl_overflow_3", "bl_single"))
    # the widest tree description reached, against the 2 087-bit worst case and the 2 560 bits
    # of a block's table
    print(f"\nhdr_bits_max {total['hdr_bits_max']}")
    assert 700 <= total["hdr_bits_max"] <= 2087


@pytest.mark.parametrize("k", range(len(E.all_cases())), ids=[c.name for c in E.all_cases()])
def test_oracle_equals_cv2_and_zlib_fed_by_rows(k):
    case, (got, e) = _cases()[k], _encoded()[k]
    ref = cv2.imencode(".png", np.ascontiguousarray(case.img[..., ::-1]))[1].tobytes()
    assert got == ref, case.name
    n = len(e.stream)
    _, zbits = P.window_bits(n)
    c = zlib.compressobj(1, zlib.DEFLATED, -zbits, 8, zlib.Z_RLE)
    rows = e.stream.tobytes()
    body = b"".join(c.compress(rows[i:i + e.rowlen]) for i in range(0, n, e.rowlen)) + c.flush()
    assert e.body == body, case.name
    assert P.adler32(e.stream) == zlib.adler32(rows)
    assert len(got) <= P.png_bound(n)


def test_every_variant_changes_an_edge_image():
    """Each one-mistake variant writes other bytes for at least one edge image; the two argued
    equivalent (png_oracle.EQUIVALENT_VARIANTS) write the same bytes for all of them."""
    files = [got for got, _ in _encoded()]
    for variant in P.VARIANTS:
        changed = [c.name for c, want in zip(_cases(), files)
                   if P.encode(c.img, variant=variant)[0] != want]
        if variant in P.EQUIVALENT_VARIANTS:
            assert not changed, (variant, changed)
        else:
            assert changed, variant


def test_the_window_never_refuses_a_cheapest_stored_block():
    """DESIGN §3.21: a block zlib's window refuses to store spans more than w - 262 bytes in at
    most 16 383 symbols, and static coding then costs less than its stored form, so `can_store`
    never decides a block type.  Checked over the blocks of the edge images and of long
    runs."""
    imgs = [c.img for c in _cases()]
    rng = np.random.default_rng(5)
    for stretch in (1, 2, 3, 258):       # 16 383 symbols of runs this long, then more
        f = np.repeat(E.noise(rng, 200000 // stretch + 1, 0), stretch)[:120001]
        f[0] = 1
        imgs.append(E.row_image(f[:len(f) - (len(f) - 1) % 3]))
    refused = 0
    for img in imgs:
        for b in P.encode(img)[1].blocks:
            if not b.can_store:
                refused += 1
                assert b.stored_len + 4 > b.static_lenb, b.stored_len
    assert refused > 0
