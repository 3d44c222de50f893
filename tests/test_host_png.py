"""The host half of the device PNG encoder: refusals, buffer sizing and its worst-case bounds,
window bits and the ABI argument checks (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

import png_oracle as P
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import png


@pytest.mark.parametrize("shape,dtype,what", [
    ((4, 4, 3), np.float32, "dtype"), ((4, 4, 3), np.uint16, "dtype"), ((4, 4), np.uint8, "shape"),
    ((4, 4, 4), np.uint8, "shape"), ((4, 4, 1), np.uint8, "shape"), ((0, 4, 3), np.uint8, "pixel"),
    ((4, 0, 3), np.uint8, "pixel"), ((1 << 15, 1 << 14, 3), np.uint8, "more than")])
def test_refusals_name_the_image(shape, dtype, what):
    with pytest.raises(ValueError, match=f"image 1: .*{what}"):
        png.Plan([((2, 2, 3), np.uint8), (shape, dtype)])


def test_window_bits_and_header_match_the_oracle():
    for n in list(range(4, 600)) + [8191, 8192, 8193, 16383, 16384, 16385, 1 << 20]:
        assert png.window_bits(n) == P.window_bits(n)
        assert bytes(png.zlib_header(n)) == P.zlib_header(n)
        assert png.deflate_bound(n) == P.deflate_bound(n) and png.png_bound(n) == P.png_bound(n)


@pytest.mark.parametrize("h,w", [(1, 1), (3, 1), (2, 2), (64, 64), (200, 300), (1, 5461)])
def test_bound_holds_for_incompressible_images(h, w):
    """Noise is the worst case zlib meets (stored and static blocks); the bound holds with room."""
    rng = np.random.default_rng(h * 1000 + w)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    data, e = P.encode(img)
    n = png.stream_length(h, w)
    assert len(e.body) <= png.deflate_bound(n) and len(data) <= png.png_bound(n)


def test_plan_layout():
    plan = png.Plan([((2, 3, 3), np.uint8), ((100, 50, 3), np.uint8), ((1, 1, 3), np.uint8)])
    d = plan.desc
    ns = [2 * 10, 100 * 151, 4]
    assert list(d[:, png.D_N]) == ns
    assert list(d[:, png.D_NTILES]) == [-(-n // png.TILE) for n in ns]
    assert list(d[:, png.D_TILE_OFF]) == [0, 1, 1 + -(-ns[1] // png.TILE)]
    assert plan.total_tiles == sum(-(-n // png.TILE) for n in ns)
    assert list(d[:, png.D_MAXBLK]) == [n // 16383 + 1 for n in ns]
    assert all(o % 16 == 0 for o in d[:, png.D_OUT_OFF])
    assert plan.max_n == ns[1] and plan.max_chunks == -(-png.zlib_bound(ns[1]) // 8192)
    for b, n in enumerate(ns):
        cmf, flg = P.zlib_header(n)
        assert (d[b, png.D_CMF], d[b, png.D_FLG]) == (cmf, flg)
        assert d[b, png.D_WBITS] == P.window_bits(n)[1]
    plan.set_sources([16, 32, 48])
    assert list(d[:, png.D_SRC]) == [16, 32, 48]


def test_abi_checks():
    lib = N.load()
    buf = C.c_void_p(16)
    args = [buf, 1, 100, 1, 1, 1, 1] + [buf] * 11 + [None]
    assert lib.mrx_png_encode(None, *args[1:]) == N.MRX_E_INVALID
    assert b"null pointer" in lib.mrx_last_error()
    bad = list(args)
    bad[1] = N.MRX_MAX_BATCH + 1
    assert lib.mrx_png_encode(*bad) == N.MRX_E_INVALID
    bad = list(args)
    bad[2] = N.MRX_PNG_MAX_STREAM + 1
    assert lib.mrx_png_encode(*bad) == N.MRX_E_INVALID
    bad = list(args)
    bad[3] = 0
    assert lib.mrx_png_encode(*bad) == N.MRX_E_INVALID
    zero = list(args)
    zero[1] = 0
    assert lib.mrx_png_encode(*zero) == N.MRX_OK
