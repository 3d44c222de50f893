"""tests/jpeg_oracle.py held bit for bit to cv2.imdecode (libjpeg-turbo) over the small cases of
the device decoder's matrix: this is what pins the formulas the device decoder restates."""
import itertools

import numpy as np
import pytest

import jpeg_inputs as JI
import jpeg_oracle as O

SMALL = [(1, 1), (1, 9), (9, 1), (2, 4), (3, 5), (7, 9), (8, 8), (15, 17), (16, 16), (17, 33)]


@pytest.mark.parametrize("samp", list(JI.SAMPLINGS))
def test_oracle_equals_cv2_small_matrix(samp):
    rng = np.random.default_rng(list(JI.SAMPLINGS).index(samp))
    for (h, w), q, kind in itertools.product(SMALL, [1, 50, 95, 100], ["smooth", "noise"]):
        blob = JI.encode(JI.image(rng, h, w, kind), q, samp)
        assert np.array_equal(O.decode(blob), JI.cv2_decode(blob)), (h, w, q, kind)


@pytest.mark.parametrize("rst,optimize,gray", [(1, False, False), (3, True, False),
                                               (64, False, True), (0, True, True)])
def test_oracle_equals_cv2_restarts_tables_gray(rst, optimize, gray):
    rng = np.random.default_rng(rst)
    for (h, w), samp in itertools.product([(7, 9), (40, 67)], ["420", "411"]):
        blob = JI.encode(JI.image(rng, h, w, "noise", gray=gray), 90, samp, rst, optimize)
        assert np.array_equal(O.decode(blob), JI.cv2_decode(blob)), (h, w, samp)


@pytest.mark.parametrize("big_endian", [False, True])
def test_oracle_orientation_equals_cv2(big_endian):
    rng = np.random.default_rng(9)
    base = JI.encode(JI.image(rng, 11, 19), 90, "420")
    for o in range(1, 9):
        blob = JI.with_exif(base, o, big_endian)
        ref = JI.cv2_decode(blob)
        got = O.decode(blob)
        assert got.shape == ref.shape and np.array_equal(got, ref), o


def test_oracle_spliced_tables_and_colour_spaces():
    rng = np.random.default_rng(10)
    base = JI.encode(JI.image(rng, 21, 30), 85, "420", rst=2)
    for blob in (JI.with_dqt16(base), JI.without_jfif_with_adobe(base, 0),
                 JI.without_jfif_with_adobe(base, 1)):
        assert np.array_equal(O.decode(blob), JI.cv2_decode(blob))


def test_oracle_idct_saturates_where_jidctint_wraps():
    """DC-only blocks (quantiser 1): pass 1's shortcut wraps at dequantised DC 8192 (8191 -> 255,
    8192 -> 0, -8193 -> 255); pass 2 clamps where jidctint.c's x & 1023 table wraps (4100 -> 513
    is 255, not 0; -4108 -> -513 is 0, not 255).  The C arithmetic is the "c" mistake."""
    q = np.ones(64, dtype=np.int64)
    for dc, want, c_want in ((8191, 255, 128), (8192, 0, 128), (-8193, 255, 128),
                             (4100, 255, 0), (-4108, 0, 255), (4000, 255, 255)):
        coef = np.zeros((1, 64), dtype=np.int64)
        coef[0, 0] = dc
        assert (O.idct_islow(coef, q) == want).all(), dc
        assert (O.idct_islow(coef, q, "c") == c_want).all(), dc


def test_oracle_refuses_corrupt_data():
    rng = np.random.default_rng(11)
    good = JI.encode(JI.image(rng, 24, 40, "noise"), 90, "420")
    with pytest.raises(ValueError, match="data ended"):
        O.decode(JI.truncated(good))
    with pytest.raises(ValueError, match="bad Huffman code"):
        O.decode(JI.with_bad_code(good))
    rst = JI.encode(JI.image(rng, 24, 40, "noise"), 90, "420", rst=1)
    with pytest.raises(ValueError, match="RST"):
        O.decode(JI.with_wrong_rst(rst))
