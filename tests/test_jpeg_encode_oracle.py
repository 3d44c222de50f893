"""The JPEG encoder's CPU restatement (jpeg_encode_oracle) against cv2.imencode('.jpg') byte for
byte over the input matrix, and the cases the matrix must reach (no GPU needed)."""
import numpy as np
import pytest

import jpeg_encode_inputs as I
import jpeg_encode_oracle as O

cv2 = pytest.importorskip("cv2")

SMALL = I.matrix(big=False)
BIG = [(n, img) for n, img in I.matrix() if n not in dict(SMALL)]


def cv2_jpeg(img, quality=95, optimize=False):
    return cv2.imencode(".jpg", np.ascontiguousarray(img[..., ::-1]),
                        [cv2.IMWRITE_JPEG_QUALITY, int(quality),
                         cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize)])[1].tobytes()


@pytest.mark.parametrize("optimize", I.OPTIMIZE)
@pytest.mark.parametrize("quality", I.QUALITIES)
def test_oracle_equals_cv2_imencode(quality, optimize):
    for name, img in SMALL:
        got, e = O.encode(img, quality, optimize)
        assert got == cv2_jpeg(img, quality, optimize), name
        assert len(got) == e.hdr + e.bytes + e.ff + 2, name


@pytest.mark.parametrize("optimize", I.OPTIMIZE)
@pytest.mark.parametrize("name", [n for n, _ in BIG])
def test_oracle_equals_cv2_imencode_large_overlays(name, optimize):
    img = dict(BIG)[name]
    assert O.encode(img, 95, optimize)[0] == cv2_jpeg(img, 95, optimize)


def test_matrix_covers_the_cases():
    """Dummy blocks right, below and in the corner; an odd chroma width in blocks; ZRL runs,
    all-EOB blocks, every AC category and 0xFF bytes to stuff."""
    shapes = {img.shape[:2] for _, img in SMALL}
    wib = {-(-w // 8) % 2 for _, w in shapes}
    hib = {-(-h // 8) % 2 for h, _ in shapes}
    assert wib == {0, 1} and hib == {0, 1}
    assert any(-(-h // 8) % 2 and -(-w // 8) % 2 for h, w in shapes)
    assert any(-(-w // 16) % 2 for _, w in shapes)
    assert {w % 16 for _, w in shapes} >= {1, 9}
    zrl = eob_only = ff = 0
    cats = set()
    for _, img in SMALL:
        for q in (50, 100):
            _, e = O.encode(img, q)
            tab, sym, _, ln = O.symbols(e.coef)
            ac = tab % 2 == 1
            zrl += int((ac & (sym == 0xF0)).sum())
            cats |= set(ln[ac & (sym != 0xF0) & (sym != 0)].tolist())
            eob_only += int((e.coef[:, 1:] == 0).all(axis=1).sum())
            ff += e.ff
    assert zrl > 0 and eob_only > 0 and ff > 0
    assert cats == set(range(1, 11))


def test_quant_tables_follow_jpeg_set_quality():
    """Quality 0 behaves as 1; 50 is the standard tables; 100 is all ones."""
    assert np.array_equal(O.quant_tables(0), O.quant_tables(1))
    assert np.array_equal(O.quant_tables(50), O.STD_QUANT)
    assert (O.quant_tables(100) == 1).all()
    assert O.quant_tables(1).max() == 255
