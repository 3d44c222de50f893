"""The PNG encoder's CPU restatement (png_oracle) against cv2.imencode('.png') byte for byte, and
its intermediates against Python's zlib where they meet (no GPU needed)."""
import zlib

import numpy as np
import pytest

import png_inputs
import png_oracle as P

cv2 = pytest.importorskip("cv2")

MATRIX = png_inputs.matrix()


@pytest.fixture(scope="module")
def encoded():
    return {name: (img, P.encode(img)) for name, img in MATRIX}


@pytest.mark.parametrize("name", [name for name, _ in MATRIX])
def test_oracle_equals_cv2_imencode(encoded, name):
    img, (got, e) = encoded[name]
    ref = cv2.imencode(".png", np.ascontiguousarray(img[..., ::-1]))[1].tobytes()
    assert got == ref
    # intermediates: the deflate body is zlib's own (level 1, Z_RLE, memLevel 8, the window cv2
    # uses), the checksum zlib's Adler-32
    n = len(e.stream)
    _, zbits = P.window_bits(n)
    c = zlib.compressobj(1, zlib.DEFLATED, -zbits, 8, zlib.Z_RLE)
    assert e.body == c.compress(e.stream.tobytes()) + c.flush()
    assert P.adler32(e.stream) == zlib.adler32(e.stream.tobytes())
    assert zlib.decompress(e.zstream) == e.stream.tobytes()
    assert len(got) <= P.png_bound(n)


def test_matrix_covers_the_cases(encoded):
    """Every window bits value, an empty final block, all three block types, and stored blocks
    after a window slide."""
    wbits = {P.window_bits(len(e.stream))[0] for _, (_, e) in encoded.values()}
    assert wbits == set(range(8, 16))
    e = encoded["sym16383"][1][1]
    assert e.nsym == 16383 and len(e.blocks) == 2 and e.blocks[-1].nsym == 0
    assert encoded["sym32766"][1][1].nsym == 32766
    types = {}
    stored_after_slide = 0
    for _, (_, e) in encoded.values():
        for b in e.blocks:
            types[b.type] = types.get(b.type, 0) + 1
            w = 1 << P.window_bits(len(e.stream))[1]
            if b.type == P.STORED and b.end > 2 * w - 262:
                stored_after_slide += 1
    print(f"\nblocks: stored {types.get(P.STORED, 0)}, static {types.get(P.STATIC, 0)}, dynamic "
          f"{types.get(P.DYNAMIC, 0)}; stored after a window slide {stored_after_slide}")
    assert all(types.get(t, 0) > 0 for t in (P.STORED, P.STATIC, P.DYNAMIC))
    assert stored_after_slide > 0


def test_parse_runs():
    """A stretch of L bytes equal to their predecessor: floor(L/258) matches of 258, then a match
    of the rest when it is at least 3, else literals."""
    for L, want in [(1, [1]), (2, [1, 1]), (3, [3]), (258, [258]), (259, [258, 1]),
                    (260, [258, 1, 1]), (261, [258, 3]), (516, [258, 258]), (520, [258, 258, 4])]:
        s = np.array([5] + [9] * (L + 1) + [4], np.uint8)     # 9 then L bytes equal to it
        sym = P.parse(s)
        codes = sym[2:2 + L]
        got = [int(c) - 256 + 3 if c >= 256 else 1 for c in codes if c >= 0]
        assert got == want, L
        assert list(sym[:2]) == [5, 9] and sym[-1] == 4


def test_trees_against_known_blocks():
    """A block of one literal kind: two 1-bit codes; the empty block: END_BLOCK alone."""
    lfreq = [0] * P.L_CODES
    lfreq[P.END_BLOCK] = 1
    b = P.block_trees(lfreq, [0] * P.D_CODES, 0, True)
    assert b.type == P.STATIC and b.static_len == 7
    lfreq[65] = 1000
    b = P.block_trees(lfreq, [0] * P.D_CODES, 1000, True)
    assert b.type == P.DYNAMIC and b.llen[65] == 1 and b.llen[P.END_BLOCK] == 1
