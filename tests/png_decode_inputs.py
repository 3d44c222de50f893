"""PNG files for the device PNG decoder's tests, written with NumPy and zlib alone (so the matrix
does not depend on which encoders a machine has), plus `cv2_decode`, the contract: cv2.imdecode
(IMREAD_COLOR) then BGR -> RGB.  A small deflate block walker (`deflate_blocks`) gives the true
block boundaries of a stream, which zlib does not expose."""
import struct
import zlib

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
COMBOS = [(ct, d) for ct in (0, 2, 3, 4, 6) for d in DEPTHS[ct]]          # all fifteen
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2),
         (0, 1, 1, 2)]                                  # (x0, y0, dx, dy) of the seven passes


def cv2_decode(blob):
    """cv2.imdecode(IMREAD_COLOR) + BGR -> RGB, or None where cv2 refuses the file."""
    import cv2

    try:
        img = cv2.imdecode(np.frombuffer(bytes(blob), np.uint8), cv2.IMREAD_COLOR)
    except cv2.error:                  # e.g. more than CV_IO_MAX_IMAGE_PIXELS
        return None
    if img is None:
        return None
    return cv2.cvtColor(img, cv2.COLOR_BGR2RGB)


def chunk(tag, data, crc=None):
    c = zlib.crc32(tag + data) if crc is None else crc
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", c & 0xFFFFFFFF)


def samples(rng, h, w, ct, depth, kind="noise", palette_size=None):
    """h x w x channels samples of `depth` bits (uint16 when depth is 16)."""
    c = CHANNELS[ct]
    top = (1 << depth) - 1 if ct != 3 else (palette_size or (1 << depth)) - 1
    if kind == "noise":
        a = rng.integers(0, top + 1, size=(h, w, c))
    elif kind == "smooth":
        y, x = np.mgrid[:h, :w]
        a = np.stack([(x * (k + 1) + y * 3 + k * 17) % (top + 1) for k in range(c)], -1)
    else:                                                  # constant
        a = np.full((h, w, c), top // 3)
    return a.astype(np.uint16 if depth == 16 else np.uint8)


def _row_bytes(a, depth):
    """The packed bytes of one row of samples (w x c)."""
    flat = a.reshape(-1).astype(np.uint32)
    if depth == 16:
        return flat.astype(">u2").tobytes()
    if depth == 8:
        return flat.astype(np.uint8).tobytes()
    per = 8 // depth
    pad = (-len(flat)) % per
    flat = np.concatenate([flat, np.zeros(pad, np.uint32)]).reshape(-1, per)
    shifts = np.array([8 - depth * (k + 1) for k in range(per)], np.uint32)
    return (flat << shifts).sum(1).astype(np.uint8).tobytes()


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def filter_rows(rows, bpp, filters):
    """Filtered stream of a pass: rows (list of bytes), each prefixed by its filter byte."""
    out = bytearray()
    prev = bytes(len(rows[0])) if rows else b""
    for r, raw in enumerate(rows):
        f = filters[r % len(filters)]
        line = bytearray(len(raw))
        for i, x in enumerate(raw):
            a = raw[i - bpp] if i >= bpp else 0
            b = prev[i]
            c = prev[i - bpp] if i >= bpp else 0
            pred = (0, a, b, (a + b) // 2, _paeth(a, b, c))[f]
            line[i] = (x - pred) & 255
        out += bytes([f]) + line
        prev = raw
    return bytes(out)


def filtered_stream(a, ct, depth, interlace=0, filters=(0, 1, 2, 3, 4)):
    """The filtered bytes of samples `a` (h x w x c): rows of each Adam7 pass, or of the image."""
    c = CHANNELS[ct]
    bpp = max(1, c * depth // 8)
    h, w = a.shape[:2]
    passes = ADAM7 if interlace else [(0, 0, 1, 1)]
    out = b""
    for x0, y0, dx, dy in passes:
        sub = a[y0::dy, x0::dx]
        if sub.shape[0] == 0 or sub.shape[1] == 0:
            continue
        out += filter_rows([_row_bytes(r, depth) for r in sub], bpp, filters)
    return out


def write(a, ct, depth, *, interlace=0, filters=(0, 1, 2, 3, 4), level=6, strategy=0, wbits=15,
          mem=8, palette=None, split=None, before=(), after=(), stream=None, extra=b"",
          trailing=b""):
    """A PNG file: IHDR, `before` chunks, PLTE (colour type 3, or when given), IDAT (split into
    chunks of `split` bytes, or one), `after` chunks, IEND.  `stream` replaces the filtered bytes
    (e.g. with too many rows); `extra` is appended to the zlib stream."""
    h, w = a.shape[:2]
    raw = filtered_stream(a, ct, depth, interlace, filters) if stream is None else stream
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, mem, strategy)
    z = co.compress(raw) + co.flush() + extra
    out = SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ct, 0, 0, interlace))
    for c in before:
        out += c
    if ct == 3 and palette is None:
        palette = default_palette(1 << depth)
    if palette is not None:
        out += chunk(b"PLTE", np.asarray(palette, np.uint8).tobytes())
    step = split or max(len(z), 1)
    for i in range(0, max(len(z), 1), step):
        out += chunk(b"IDAT", z[i:i + step])
    for c in after:
        out += c
    return out + chunk(b"IEND", b"") + trailing


def default_palette(n, seed=7):
    return np.random.default_rng(seed).integers(0, 256, size=(n, 3))


def exif_chunk(orientation, big_endian=False):
    e = ">" if big_endian else "<"
    tiff = (b"MM" if big_endian else b"II") + struct.pack(e + "HI", 42, 8)
    tiff += struct.pack(e + "H", 1) + struct.pack(e + "HHIHH", 0x0112, 3, 1, orientation, 0)
    tiff += struct.pack(e + "I", 0)
    return chunk(b"eXIf", tiff)


def chunks(blob):
    """[(tag, start of the length field, data start, data length)] of a file."""
    out, p = [], 8
    while p + 8 <= len(blob):
        n = struct.unpack(">I", blob[p:p + 4])[0]
        out.append((blob[p + 4:p + 8], p, p + 8, n))
        p += 12 + n
    return out


def replace_chunk(blob, tag, fn):
    """The file with the first `tag` chunk replaced by fn(start, data start, length) bytes."""
    for t, s, d, n in chunks(blob):
        if t == tag:
            return blob[:s] + fn(blob, s, d, n) + blob[d + n + 4:]
    raise KeyError(tag)


def zlib_stream(blob):
    return b"".join(blob[d:d + n] for t, _, d, n in chunks(blob) if t == b"IDAT")


def with_zlib_stream(blob, z, split=None):
    """The file with its IDAT chunks replaced by one (or `split`-byte) chunks of z."""
    cs = chunks(blob)
    first = next(s for t, s, _, _ in cs if t == b"IDAT")
    last = max(d + n + 4 for t, _, d, n in cs if t == b"IDAT")
    step = split or len(z)
    idat = b"".join(chunk(b"IDAT", z[i:i + step]) for i in range(0, len(z), step))
    return blob[:first] + idat + blob[last:]


class _Bits:
    def __init__(self, data, pos=0):
        self.data, self.pos = data, pos

    def get(self, n):
        v = 0
        for k in range(n):
            byte = self.data[(self.pos + k) >> 3]
            v |= ((byte >> ((self.pos + k) & 7)) & 1) << k
        self.pos += n
        return v


def _canonical(lengths):
    """{(length, code): symbol} of a canonical Huffman code."""
    counts = [0] * 16
    for l in lengths:
        counts[l] += 1
    counts[0] = 0
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + counts[b - 1]) << 1
        nxt[b] = code
    out = {}
    for s, l in enumerate(lengths):
        if l:
            out[(l, nxt[l])] = s
            nxt[l] += 1
    return out


def _sym(bits, table):
    code, length = 0, 0
    while True:
        code = (code << 1) | bits.get(1)
        length += 1
        if (length, code) in table:
            return table[(length, code)]
        if length > 15:
            raise ValueError("bad code")


LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
         131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DEXT = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
         2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577]
ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def deflate_blocks(z):
    """[(first bit in the deflate stream, output offset, type, final)] of every block of a zlib
    stream z (valid streams only; slow, for small files)."""
    bits = _Bits(z[2:])
    out, blocks = 0, []
    fixed_l = _canonical([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
    fixed_d = _canonical([5] * 30)
    while True:
        start = bits.pos
        final, typ = bits.get(1), bits.get(2)
        blocks.append((start, out, typ, final))
        if typ == 0:
            bits.pos = (bits.pos + 7) & ~7
            n = bits.get(16)
            bits.get(16)
            bits.pos += 8 * n
            out += n
        else:
            if typ == 1:
                lt, dt = fixed_l, fixed_d
            else:
                hlit, hdist, hclen = bits.get(5) + 257, bits.get(5) + 1, bits.get(4) + 4
                cl = [0] * 19
                for k in range(hclen):
                    cl[ORDER[k]] = bits.get(3)
                ct = _canonical(cl)
                lens = []
                while len(lens) < hlit + hdist:
                    s = _sym(bits, ct)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + bits.get(2))
                    elif s == 17:
                        lens += [0] * (3 + bits.get(3))
                    else:
                        lens += [0] * (11 + bits.get(7))
                lt, dt = _canonical(lens[:hlit]), _canonical(lens[hlit:])
            while True:
                s = _sym(bits, lt)
                if s < 256:
                    out += 1
                elif s == 256:
                    break
                else:
                    out += LBASE[s - 257] + bits.get(LEXT[s - 257])
                    d = _sym(bits, dt)
                    bits.get(DEXT[d])
        if final:
            return blocks
