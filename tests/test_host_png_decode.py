"""The host half of the device PNG decoder: chunk parse, refusals (each one also refused by
cv2.imdecode on the same bytes), files libpng only warns about, buffer sizing, routing by
signature and the ABI argument checks (no GPU needed)."""
import ctypes as C
import struct
import zlib

import numpy as np
import pytest

import jpeg_inputs as JI
import png_decode_inputs as P
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import exif, imagefile, jpeg, png


def _img(h=20, w=17, ct=2, depth=8, seed=0):
    return P.samples(np.random.default_rng(seed), h, w, ct, depth)


def _good(**kw):
    return P.write(_img(), 2, 8, **kw)


def _stored(data, final):
    return bytes([final]) + struct.pack("<HH", len(data), 0xFFFF ^ len(data)) + data


def test_parse_known_answers():
    hd = png.parse(_good())
    assert (hd.height, hd.width, hd.color_type, hd.depth, hd.interlace) == (20, 17, 2, 8, 0)
    assert hd.filtered == 20 * (1 + 51) and hd.orientation == 1 and hd.shape == (20, 17, 3)
    assert hd.window == 1 << 15 and len(hd.idat) == 1
    hd = png.parse(P.write(_img(5, 6, 0, 2), 0, 2, interlace=1, wbits=9, split=3))
    assert hd.filtered == png.filtered_length(5, 6, 0, 2, 1) == len(
        P.filtered_stream(_img(5, 6, 0, 2), 0, 2, 1))
    assert hd.window == 512 and len(hd.idat) == -(-len(P.zlib_stream(P.write(
        _img(5, 6, 0, 2), 0, 2, interlace=1, wbits=9))) // 3)
    pal = P.default_palette(10)
    hd = png.parse(P.write(_img(4, 4, 3, 4), 3, 4, palette=pal))
    assert hd.palette_len == 10 and np.array_equal(hd.palette[:10], pal)
    for o in range(1, 9):
        for where in ("before", "after"):
            hd = png.parse(_good(**{where: [P.exif_chunk(o, big_endian=o % 2 == 0)]}))
            assert hd.orientation == o
            assert hd.shape == ((17, 20, 3) if o >= 5 else (20, 17, 3))


@pytest.mark.parametrize("ct,depth", P.COMBOS)
@pytest.mark.parametrize("interlace", [0, 1])
def test_filtered_length_matches_the_writer(ct, depth, interlace):
    for h, w in [(1, 1), (3, 5), (8, 8), (9, 13)]:
        a = _img(h, w, ct, depth)
        assert png.filtered_length(h, w, ct, depth, interlace) == len(
            P.filtered_stream(a, ct, depth, interlace))


def _refusals():
    g = _good()
    z = P.zlib_stream(g)
    raw = P.filtered_stream(_img(), 2, 8)
    idat_crc = P.replace_chunk(g, b"IDAT", lambda b, s, d, n: b[s:d + n] + bytes(4))
    out = [
        ("signature", b"\x89PNG\r\n\x1a\x0b" + g[8:], "signature"),
        ("IHDR crc", P.replace_chunk(g, b"IHDR", lambda b, s, d, n: b[s:d + n] + bytes(4)),
         "IHDR"),
        ("no IEND", g[:-12], "IEND"),
        ("unknown critical", g[:33] + P.chunk(b"QRST", b"x") + g[33:], "critical"),
        ("width", P.replace_chunk(g, b"IHDR", lambda b, s, d, n: P.chunk(
            b"IHDR", struct.pack(">IIBBBBB", 1000001, 20, 8, 2, 0, 0, 0))), "size"),
        ("bad depth", P.replace_chunk(g, b"IHDR", lambda b, s, d, n: P.chunk(
            b"IHDR", struct.pack(">IIBBBBB", 17, 20, 4, 2, 0, 0, 0))), "colour type"),
        ("pixels", P.replace_chunk(g, b"IHDR", lambda b, s, d, n: P.chunk(
            b"IHDR", struct.pack(">IIBBBBB", 40000, 30000, 1, 0, 0, 0, 0))), "pixels"),
        ("CINFO 8", P.with_zlib_stream(g, bytes([0x88, 0x1c]) + z[2:]), "window size"),
        ("FDICT", P.with_zlib_stream(g, bytes([0x78, 0x20 | (31 - (0x7820 % 31))]) + z[2:]),
         "dictionary"),
        ("FCHECK", P.with_zlib_stream(g, bytes([0x78, 0x9d]) + z[2:]), "header check"),
        ("interrupted IDAT", g[:33] + P.chunk(b"IDAT", z[:9]) + P.chunk(b"tEXt", b"a\x00b") +
         P.chunk(b"IDAT", z[9:]) + P.chunk(b"IEND", b""), "consecutive"),
        ("APNG", g[:33] + P.chunk(b"acTL", bytes(8)) + g[33:], "APNG"),
        ("no PLTE", P.replace_chunk(P.write(_img(4, 4, 3, 8), 3, 8), b"PLTE",
                                    lambda b, s, d, n: b""), "PLTE"),
        ("empty PLTE in an RGB file", P.replace_chunk(
            P.write(_img(), 2, 8, palette=np.zeros((1, 3))), b"PLTE",
            lambda b, s, d, n: P.chunk(b"PLTE", b"")), "PLTE length 0"),
        ("PLTE of 4 bytes", P.replace_chunk(P.write(_img(4, 4, 3, 8), 3, 8), b"PLTE",
                                            lambda b, s, d, n: P.chunk(b"PLTE", bytes(4))),
         "PLTE length 4"),
    ]
    return out, idat_crc, raw


@pytest.mark.parametrize("k", range(15))
def test_refusals_name_the_index_and_cv2_refuses_too(k):
    cases, _, _ = _refusals()
    name, blob, why = cases[k]
    assert P.cv2_decode(blob) is None, name
    with pytest.raises(png.PngError, match=f"image 7: .*{why}"):
        png.parse(blob, 7)
    with pytest.raises(ValueError, match="image 7"):
        png.DecodePlan([_good(), blob], index=[6, 7])


def test_device_refusals_are_refused_by_cv2():
    """What only the device finds (the image data) is refused by cv2 as well; the host accepts
    the header (tests/test_gpu_png_decode.py checks the device's status)."""
    for name, blob in corrupt_data_cases():
        assert P.cv2_decode(blob) is None, name
        png.parse(blob)


def corrupt_data_cases():
    g = _good()
    z = P.zlib_stream(g)
    raw = P.filtered_stream(_img(), 2, 8)
    bad = bytearray(raw)
    bad[52] = 5
    return [
        ("IDAT crc", P.replace_chunk(g, b"IDAT", lambda b, s, d, n: b[s:d + n] + bytes(4))),
        ("adler exact", P.with_zlib_stream(g, z[:-1] + bytes([z[-1] ^ 1]))),
        ("truncated", P.with_zlib_stream(g, z[:len(z) // 2])),
        ("no trailer", P.with_zlib_stream(g, z[:-4])),
        ("filter 5", P.write(_img(), 2, 8, stream=bytes(bad))),
        ("invalid block type", P.with_zlib_stream(g, b"\x78\x01" + b"\x07" + bytes(8))),
        ("invalid block after the rows", P.with_zlib_stream(
            g, b"\x78\x01" + _stored(raw, 0) + b"\x07" + bytes(8))),
        ("stored NLEN", P.with_zlib_stream(g, b"\x78\x01\x01" + struct.pack("<HH", 5, 5) +
                                           bytes(5))),
        ("too far back", P.with_zlib_stream(g, b"\x78\x01" + _fixed_match_first() + bytes(8))),
        ("short final block", P.with_zlib_stream(g, b"\x78\x01" + _stored(raw[:-1], 1) +
                                                 struct.pack(">I", zlib.adler32(raw[:-1])))),
    ]


def _fixed_match_first():
    """A fixed-code block whose first symbol is a match of length 3 at distance 1 (nothing to
    copy from)."""
    bits = [1, 1, 0]                     # final, BTYPE = 01 (LSB first)
    bits += [0, 0, 0, 0, 0, 0, 1]        # length code 257 (7 bits, MSB first)
    bits += [0, 0, 0, 0, 0]              # distance code 0
    bits += [0] * 7                      # end of block
    out = bytearray((len(bits) + 7) // 8)
    for i, v in enumerate(bits):
        out[i >> 3] |= v << (i & 7)
    return bytes(out)


def warning_cases():
    """Files libpng reads with a warning: each decodes to the undamaged image."""
    a = _img()
    g = P.write(a, 2, 8)
    raw = P.filtered_stream(a, 2, 8)
    big = P.write(a, 2, 8, stream=raw + bytes(200))
    zb = P.zlib_stream(big)
    return [
        ("ancillary crc", P.write(a, 2, 8, before=[P.chunk(b"tEXt", b"a\x00b", crc=1)])),
        ("exif crc ignored", P.write(a, 2, 8, before=[P.exif_chunk(3)[:-4] + bytes(4)])),
        ("extra compressed data", P.write(a, 2, 8, extra=b"junkjunk")),
        ("too much image data", big),
        ("too much, bad adler", P.with_zlib_stream(big, zb[:-1] + bytes([zb[-1] ^ 1]))),
        ("idat split at every byte", P.write(a, 2, 8, split=1)),
        ("bytes after IEND", g + b"trailing"),
        ("PLTE in a gray file", P.write(_img(20, 17, 0, 8), 0, 8, palette=P.default_palette(5))),
        ("PLTE of 4 bytes in an RGB file", P.replace_chunk(
            P.write(a, 2, 8, palette=np.zeros((1, 3))), b"PLTE",
            lambda b, s, d, n: P.chunk(b"PLTE", b"\x01\x02\x03\x04"))),
        ("two eXIf chunks: the first counts", P.write(a, 2, 8, before=[P.exif_chunk(1)],
                                                      after=[P.exif_chunk(3)])),
    ]


def ancillary_cases():
    """tRNS, gAMA and sBIT change nothing: (name, file with the chunk, file without)."""
    rng = np.random.default_rng(9)
    out = []
    for ct, depth, trns in [(0, 8, b"\x00\x05"), (0, 16, b"\x12\x34"), (2, 8, bytes(6)),
                            (2, 16, bytes(6)), (3, 8, b"\x00\x80"), (3, 2, b"\x10"),
                            (4, 8, None), (6, 16, None)]:
        x = P.samples(rng, 11, 13, ct, depth)
        base = P.write(x, ct, depth)
        ip = next(s for t, s, _, _ in P.chunks(base) if t == b"IDAT")
        nbit = 1 if ct in (0, 3) else 2 if ct == 4 else 3 if ct == 2 else 4
        extra = [P.chunk(b"gAMA", struct.pack(">I", 45455)),
                 P.chunk(b"sBIT", bytes([min(depth, 8) - 1 or 1] * nbit))]
        if trns is not None:
            extra.append(P.chunk(b"tRNS", trns))
        for c in extra:
            out.append((f"{c[4:8].decode()} ct{ct} d{depth}", base[:ip] + c + base[ip:], base))
    return out


def test_ancillary_chunks_change_nothing_in_cv2():
    for name, blob, base in ancillary_cases():
        assert np.array_equal(P.cv2_decode(blob), P.cv2_decode(base)), name
        assert png.parse(blob).shape == png.parse(base).shape


def _bits(bits, pad=8):
    out = bytearray((len(bits) + 7) // 8 + pad)
    for i, v in enumerate(bits):
        out[i >> 3] |= v << (i & 7)
    return bytes(out)


def _msb(v, n):
    return [(v >> (n - 1 - k)) & 1 for k in range(n)]


LIT0 = _msb(0x30, 8)                 # fixed code of literal 0
LEN3 = _msb(1, 7)                    # fixed code 257: length 3


def after_the_rows_cases():
    """Errors in the deflate stream past the image's last row, as cv2 reads them with the stream
    in one IDAT chunk, in 1-byte and in 7-byte chunks: (name, blob, [decodes? per chunking]).
    libpng has every row once it needs a byte past them; an error it meets before that is fatal
    when it comes in the same chunk as the last row, so the outcome depends on the chunking."""
    a = _img()
    g = P.write(a, 2, 8)
    raw = P.filtered_stream(a, 2, 8)
    rows = b"\x78\x01" + _stored(raw, 0)
    far = LEN3 + _msb(29, 5) + [0] * 13             # distance 24577, past the stream start
    return [
        ("invalid block type after one more byte", b"\x78\x01" + _stored(raw + b"\x00", 0) +
         b"\x07" + bytes(8), [True, True, True]),
        ("invalid code after one more byte", rows + _fixed_literal_then_code(286),
         [True, True, True]),
        ("distance too far back at the last row", rows + _bits([0, 1, 0] + far), [True] * 3),
        ("distance too far back after one more byte", rows + _bits([0, 1, 0] + LIT0 + far),
         [True] * 3),
        ("invalid block type at the last row", rows + b"\x07" + bytes(8), [False, True, False]),
        ("invalid code at the last row", rows + _bits([0, 1, 0] + _msb(0xC6, 8)),
         [False, True, False]),
        ("invalid distance code at the last row", rows + _bits([0, 1, 0] + LEN3 + _msb(30, 5)),
         [False, True, False]),
        ("no trailer after one more byte", rows + _bits([1, 1, 0] + LIT0 + [0] * 7, 0),
         [False, True, False]),
    ]


def device_accepts(outcomes):
    """The device decodes what cv2 decodes however the data is chunked, and refuses the rest."""
    return all(outcomes)


def test_errors_after_the_rows_as_cv2_reads_them():
    ref = P.cv2_decode(P.write(_img(), 2, 8))
    g = P.write(_img(), 2, 8)
    for name, z, outcomes in after_the_rows_cases():
        for split, decodes in zip((None, 1, 7), outcomes):
            got = P.cv2_decode(P.with_zlib_stream(g, z, split))
            assert (got is not None) == decodes, (name, split)
            if decodes:
                assert np.array_equal(got, ref), (name, split)
        png.parse(P.with_zlib_stream(g, z))


def _fixed_literal_then_code(code):
    """A non-final fixed-code block: literal 0 then a literal/length code (e.g. 286, invalid)."""
    bits = [0, 1, 0]
    bits += [0, 0, 1, 1, 0, 0, 0, 0]                        # literal 0: 00110000
    v = 0xC0 + (code - 280)                                 # codes 280..287: 8 bits from 11000000
    bits += [(v >> (7 - k)) & 1 for k in range(8)]
    out = bytearray((len(bits) + 7) // 8 + 8)
    for i, b in enumerate(bits):
        out[i >> 3] |= b << (i & 7)
    return bytes(out)


def test_warning_cases_are_accepted_and_cv2_decodes_them():
    ref = P.cv2_decode(P.write(_img(), 2, 8))
    for name, blob in warning_cases():
        got = P.cv2_decode(blob)
        assert got is not None, name
        if "gray" not in name:
            assert np.array_equal(got, ref), name
        if "eXIf" in name:
            assert png.parse(blob).orientation == 1
        png.parse(blob)


def test_plan_sizes_depend_on_headers_and_lengths_only():
    rng = np.random.default_rng(3)
    a = [P.write(P.samples(rng, 30, 40, 6, 16), 6, 16, level=0),
         P.write(P.samples(rng, 9, 70, 3, 2), 3, 2, interlace=1, level=0)]
    b = [P.write(P.samples(rng, 30, 40, 6, 16), 6, 16, level=0),
         P.write(P.samples(rng, 9, 70, 3, 2), 3, 2, interlace=1, level=0)]
    assert [len(x) for x in a] == [len(x) for x in b]
    pa, pb = png.DecodePlan(a), png.DecodePlan(b)
    assert np.array_equal(pa.desc, pb.desc) and np.array_equal(pa.chunks, pb.chunks)
    for k in ("z_bytes", "filt_bytes", "block_words", "max_n", "max_pixels", "n_chunks",
              "max_zlen", "max_tiles", "total_tiles", "max_blocks"):
        assert getattr(pa, k) == getattr(pb, k), k
    assert pa.max_n == png.filtered_length(30, 40, 6, 16, 0)
    d = pa.desc
    assert d[1, png.DD_FILT_OFF] >= d[0, png.DD_N] and d[1, png.DD_Z_OFF] >= d[0, png.DD_Z_LEN]


def test_exif_parser_is_shared():
    tiff = P.exif_chunk(6)[8:-4]
    assert exif.orientation(tiff) == 6
    assert jpeg._exif_orientation(b"Exif\x00\x00" + tiff) == 6


def test_routing_by_signature():
    p = _good()
    j = JI.encode(JI.image(np.random.default_rng(0), 8, 8))
    assert imagefile.kind(p) == "png" and imagefile.kind(j) == "jpeg"
    with pytest.raises(ValueError, match="image 3: neither a JPEG nor a PNG file"):
        imagefile.kind(b"GIF89a", 3)
    assert imagefile.shape(p) == (20, 17, 3)
    plans, shapes, kinds = imagefile.plan_batch([j, p, j, p], index=[4, 5, 6, 7])
    assert kinds == ["jpeg", "png", "jpeg", "png"]
    assert shapes == [(8, 8, 3), (20, 17, 3), (8, 8, 3), (20, 17, 3)]
    assert sorted(pos for _, ps in plans for pos in ps) == [0, 1, 2, 3]
    with pytest.raises(jpeg.JpegError, match="not a JPEG"):
        jpeg.Plan([p])


def test_abi_argument_checks():
    lib = N.load()
    p = C.c_void_p(16)
    null = C.c_void_p(0)
    args = [p, p, p, p, 1, 1, 1024, 64, 100, 1, 1, 17, 4] + [p] * 11 + [null]
    assert lib.mrx_png_decode(null, *args[1:]) == N.MRX_E_INVALID
    assert lib.mrx_png_decode(*args[:15], null, *args[16:]) == N.MRX_E_INVALID
    for k, v in [(4, N.MRX_MAX_BATCH + 1), (4, -1), (5, 0), (6, 1),
                 (6, N.MRX_PNG_DEC_MAX_FILTERED + 1), (7, 0), (7, (1 << 30) + 1), (8, 1),
                 (8, N.MRX_PNG_DEC_MAX_FILE + 1), (9, 0), (10, 0), (11, 0), (12, -1),
                 (12, N.MRX_PNG_DEC_MAX_SLOTS + 1)]:
        a = list(args)
        a[k] = v
        assert lib.mrx_png_decode(*a) == N.MRX_E_INVALID, (k, v)
        assert b"mrx_png_decode" in lib.mrx_last_error()
    a = list(args)
    a[4], a[5] = 0, 0
    assert lib.mrx_png_decode(*a) == N.MRX_OK          # zero images: nothing launched
