"""The host half of the device JPEG decoder: header parse, refusals, Huffman tables, buffer sizing
and the ABI argument checks (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

import jpeg_inputs as JI
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import jpeg


def _blob(h=40, w=67, **kw):
    return JI.encode(JI.image(np.random.default_rng(0), h, w), **kw)


def test_parse_known_answers():
    hd = jpeg.parse(_blob(40, 67, sampling="420", rst=3))
    assert (hd.height, hd.width, hd.ncomp, hd.color) == (40, 67, 3, jpeg.COLOR_YCC)
    assert hd.samp == [(2, 2), (1, 1), (1, 1)] and (hd.hmax, hd.vmax) == (2, 2)
    assert (hd.mcux, hd.mcuy, hd.bpm, hd.restart_interval) == (5, 3, 6, 3)
    assert hd.orientation == 1 and hd.shape == (40, 67, 3)
    assert jpeg.parse(_blob(sampling="411")).samp == [(4, 1), (1, 1), (1, 1)]
    assert jpeg.parse(_blob(sampling="440")).samp == [(1, 2), (1, 1), (1, 1)]
    g = jpeg.parse(JI.encode(JI.image(np.random.default_rng(0), 9, 9, gray=True)))
    assert g.ncomp == 1 and g.color == jpeg.COLOR_GRAY and g.bpm == 1
    assert jpeg.parse(JI.without_jfif_with_adobe(_blob(), 0)).color == jpeg.COLOR_RGB
    assert jpeg.parse(JI.without_jfif_with_adobe(_blob(), 1)).color == jpeg.COLOR_YCC
    q8 = jpeg.parse(_blob()).tables[0][2]
    assert np.array_equal(jpeg.parse(JI.with_dqt16(_blob())).tables[0][2], q8)


@pytest.mark.parametrize("o", range(1, 9))
def test_exif_orientation_and_shape(o):
    hd = jpeg.parse(JI.with_exif(_blob(40, 67), o, big_endian=o % 2 == 0))
    assert hd.orientation == o
    assert hd.shape == ((67, 40, 3) if o >= 5 else (40, 67, 3))


def test_huffman_tables_match_canonical_codes():
    hd = jpeg.parse(_blob(optimize=True))
    for dc, ac, _ in hd.tables:
        for t in (dc, ac):
            code, k = 0, 0
            for length in range(1, 17):
                for _ in range(t.bits[length - 1]):
                    if length <= jpeg.FAST_BITS:
                        e = int(t.lookup[code << (jpeg.FAST_BITS - length)])
                        assert (e >> 8, e & 255) == (length, t.vals[k])
                    else:
                        assert code <= t.maxcode[length]
                        assert t.vals[t.valptr[length] + code] == t.vals[k]
                    code += 1
                    k += 1
                code <<= 1


def _patch(blob, marker, fn):
    for code, s, e in JI.segments(blob):
        if code == marker:
            return blob[:s] + fn(blob[s:e]) + blob[e:]
    raise AssertionError


@pytest.mark.parametrize("make,reason", [
    (lambda: b"\x89PNG\r\n\x1a\n" + bytes(64), "not a JPEG file"),
    (lambda: _blob(progressive=True), "progressive"),
    (lambda: _patch(_blob(), 0xC0, lambda s: s[:1] + b"\xc3" + s[2:]), "lossless"),
    (lambda: _patch(_blob(), 0xC0, lambda s: s[:1] + b"\xc9" + s[2:]), "arithmetic"),
    (lambda: _patch(_blob(), 0xC0, lambda s: s[:1] + b"\xc5" + s[2:]), "hierarchical"),
    (lambda: _patch(_blob(), 0xC0, lambda s: s[:4] + b"\x0c" + s[5:]), "12-bit"),
    (lambda: _patch(_blob(), 0xC0, lambda s: s[:5] + b"\x00\x00" + s[7:]), "DNL"),
    (lambda: _blob()[:30], "truncated"),
    (lambda: _patch(_blob(), 0xC4, lambda s: s[:2] + b"\x00\x03" + s[4:5]), "Huffman table"),
    (lambda: _patch(_blob(), 0xDA, lambda s: s[:6] + b"\x77" + s[7:]), "missing Huffman table"),
    (lambda: _patch(_blob(), 0xC0, lambda s: s[:12] + b"\x03" + s[13:]),
     "missing quantisation table"),
    (lambda: _patch(_blob(), 0xC0, lambda s: s[:11] + b"\x44" + s[12:]), "blocks per MCU"),
    (lambda: _patch(_blob(), 0xC0, lambda s: s[:11] + b"\x32" + s[12:14] + b"\x22" + s[15:]),
     "non-integral"),
    (lambda: _patch(_blob(), 0xDA, lambda s: s[:4] + b"\x01" + s[5:]), "non-interleaved"),
    (lambda: _patch(_blob(), 0xC0, lambda s: s[:5] + b"\x9c\x40\x9c\x40" + s[9:]),
     "more than 1073741824 pixels"),
    (lambda: _blob()[:JI.scan_start(_blob())] + b"\xff\xd9", "data ended before the last MCU"),
    (lambda: _blob()[:JI.scan_start(_blob()) + 10] + b"\xff\xd9",
     "data ended before the last MCU"),
])
def test_refusals_name_the_image_and_reason(make, reason):
    good = _blob()
    with pytest.raises(ValueError, match="image 1: .*" + reason):
        jpeg.Plan([good, make()])


def test_size_refusals_agree_with_cv2():
    """A header claiming 40000 x 40000 pixels is refused before any buffer is sized, as
    cv2.imdecode refuses it (CV_IO_MAX_IMAGE_PIXELS); a scan with no room for its blocks too."""
    import cv2

    big = _patch(_blob(), 0xC0, lambda s: s[:5] + b"\x9c\x40\x9c\x40" + s[9:])
    with pytest.raises(cv2.error, match="CV_IO_MAX_IMAGE_PIXELS"):
        JI.cv2_decode(big)
    with pytest.raises(ValueError, match="pixels"):
        jpeg.Plan([big])
    at_limit = _patch(_blob(), 0xC0, lambda s: s[:5] + b"\x80\x00\x80\x00" + s[9:])
    with pytest.raises(ValueError, match="data ended"):    # 2^30 pixels: only the scan is short
        jpeg.Plan([at_limit])


def test_refusal_of_bad_types_and_S():
    with pytest.raises(TypeError, match="image 0"):
        jpeg.Plan(["not bytes"])
    with pytest.raises(ValueError, match="S=48"):
        jpeg.Plan([_blob()], 48)


def test_buffer_sizes_follow_headers_and_file_lengths():
    blobs = [_blob(40, 67, rst=3), _blob(16, 16), bytearray(_blob(9, 9, sampling="444"))]
    plan = jpeg.Plan([memoryview(bytes(b)) for b in blobs], 64)
    assert plan.B == 3 and plan.shapes == [(40, 67, 3), (16, 16, 3), (9, 9, 3)]
    units = [5, 1, 1]
    assert plan.units == sum(units) and list(plan.unit_img) == [0] * 5 + [1, 2]
    d = plan.desc
    for b, blob in enumerate(blobs):
        scan = len(blob) - d[b, jpeg.D_SCAN_OFF]
        assert d[b, jpeg.D_NUNITS] == units[b]
        assert d[b, jpeg.D_SUB_CAP] == -(-scan * 8 // 64) + units[b]
        assert d[b, jpeg.D_FILE_LEN] == len(blob)
        o = d[b, jpeg.D_FILE_OFF]
        assert plan.files[o:o + len(blob)].tobytes() == bytes(blob)
    assert list(d[:, jpeg.D_NBLOCKS]) == [15 * 6, 1 * 6, 4 * 3]
    assert list(d[:, jpeg.D_COEF_OFF]) == [0, 90, 96] and plan.coef_blocks == 108
    assert plan.unst_bytes >= sum(len(b) - d[b_, jpeg.D_SCAN_OFF] + 8 for b_, b in enumerate(blobs))
    assert plan.max_subs == int(d[:, jpeg.D_SUB_CAP].max())


def _lib():
    return N.load()


def test_abi_argument_checks():
    lib = _lib()
    p = C.c_void_p(16)
    null = C.c_void_p(0)
    args = [p, p, p, p, 1, 1, 1024, 1, p, p, p, 1, p, null]
    assert lib.mrx_jpeg_coefficients(*args[:3], null, *args[4:]) == -1
    for S in (0, 16, 48, 65568):
        a = list(args)
        a[6] = S
        assert lib.mrx_jpeg_coefficients(*a) == -1
        assert b"S=" in lib.mrx_last_error()
    a = list(args)
    a[4] = N.MRX_MAX_BATCH + 1
    assert lib.mrx_jpeg_coefficients(*a) == -1
    a = list(args)
    a[7] = 0
    assert lib.mrx_jpeg_coefficients(*a) == -1
    a = list(args)
    a[4], a[5] = 0, 0
    assert lib.mrx_jpeg_coefficients(*a) == 0          # zero images: nothing launched
    pargs = [p, p, p, p, 1, 1, 1, p, p, p, null]
    assert lib.mrx_jpeg_pixels(null, *pargs[1:]) == -1
    a = list(pargs)
    a[6] = 0
    assert lib.mrx_jpeg_pixels(*a) == -1
    a = list(pargs)
    a[4] = 0
    assert lib.mrx_jpeg_pixels(*a) == 0
