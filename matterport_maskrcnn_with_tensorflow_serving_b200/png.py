"""Host halves of the device PNG encoder (csrc/png.cu, `mrx_png_encode`) and decoder
(csrc/png_decode.cu, `mrx_png_decode`).

NumPy only.  `Plan` checks each image and lays the batch out from the images' sizes alone: the
filtered stream length n = H * (3W + 1), the window bits cv2 writes into the zlib header, every
device buffer's offsets and a worst-case bound on each file, so that every buffer is sized before
anything runs.  What is encoded is what `cv2.imwrite(path, rgb[..., ::-1])` writes for a uint8
H x W x 3 RGB image (tests/png_oracle.py states how); anything else raises ValueError naming the
image's index.

`parse` walks a file's chunks (never the image data) and `DecodePlan` lays a batch of files out
for the decoder from the headers and file lengths alone.  What is accepted decodes bit for bit as
`cv2.imdecode(buf, IMREAD_COLOR)` then BGR -> RGB: every colour type and bit depth, Adam7, EXIF
orientation from an eXIf chunk before or after the image data.  Anything else raises `PngError`
(a ValueError) naming the image's index and the reason: what libpng refuses, APNG files (cv2
decodes those through its own animation path), and a few files libpng reads with a warning whose
outcome depends on how the data is chunked (see `parse`).
"""
from __future__ import annotations

import struct
import zlib

import numpy as np

from . import exif

TILE = 2048                       # stream positions per tile of the device scans
SYMS_PER_BLOCK = 16383            # deflate symbols per block (zlib's lit_bufsize - 1)
IDAT_BYTES = 8192                 # libpng's zlib buffer: the data bytes of every full IDAT chunk
MAX_STREAM = 1 << 30              # mrx.h MRX_PNG_MAX_STREAM: positions stay in int32
BLK_TAB_WORDS = 654               # int32 per block: frequencies, codes, tree description
BLK_INFO_WORDS = 8
IMG_INFO_WORDS = 8

# ---- the device descriptor: int64 words per image (csrc/png.cu, D_*) ----
(D_SRC, D_H, D_W, D_N, D_STREAM_OFF, D_TILE_OFF, D_NTILES, D_STRETCH_OFF, D_STRETCH_CAP,
 D_BLK_OFF, D_MAXBLK, D_BLKPOS_OFF, D_ZBUF_OFF, D_OUT_OFF, D_WBITS, D_CMF, D_FLG) = range(17)
DESC_WORDS = 20

BLOCK_TYPES = ("stored", "static", "dynamic")


def stream_length(h, w):
    """Filtered bytes of an h x w image: one filter byte and 3w sample bytes per row."""
    return h * (3 * w + 1)


def window_bits(n):
    """(window bits in the zlib header, windowBits zlib compresses with) for n filtered bytes:
    libpng shrinks the window while the whole stream fits in half of it; zlib's smallest is 9."""
    wb, half = 15, 16384
    while n <= half and wb > 8:
        half >>= 1
        wb -= 1
    return wb, max(wb, 9)


def zlib_header(n):
    """CMF and FLG: deflate with the header window bits, FLEVEL 0, FCHECK."""
    wb, _ = window_bits(n)
    cmf = ((wb - 8) << 4) | 8
    return cmf, 31 - (cmf << 8) % 31


def max_blocks(n):
    """Deflate blocks of an n-byte stream at most: one per 16383 symbols, plus the final one."""
    return n // SYMS_PER_BLOCK + 1


def deflate_bound(n):
    """Worst-case deflate bytes for n filtered bytes.  zlib never picks a block larger than its
    static coding (at most 9 bits a byte plus the 3-bit header and a 7-bit end code) and a stored
    block takes 8 bits a byte plus at most 42; there are at most n // 16383 + 2 blocks."""
    return (9 * n + 42 * (n // SYMS_PER_BLOCK + 2) + 7) // 8


def zlib_bound(n):
    return 2 + deflate_bound(n) + 4


def png_bound(n):
    """Worst-case file bytes: signature and IHDR (33), the IDAT chunks (12 bytes each around at
    most 8192 zlib bytes) and IEND (12)."""
    z = zlib_bound(n)
    return 33 + z + 12 * (-(-z // IDAT_BYTES)) + 12


def check_image(shape, dtype, index):
    """Refuse what the device encoder does not write as cv2.imwrite would: anything but uint8
    H x W x 3 with H, W >= 1 and a filtered stream of at most MAX_STREAM bytes."""
    if np.dtype(dtype) != np.uint8:
        raise ValueError(f"image {index}: dtype {np.dtype(dtype)} (expected uint8)")
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"image {index}: shape {tuple(shape)} (expected H x W x 3 RGB)")
    h, w = int(shape[0]), int(shape[1])
    if h == 0 or w == 0:
        raise ValueError(f"image {index}: {h}x{w} has no pixel")
    n = stream_length(h, w)
    if n > MAX_STREAM:
        raise ValueError(f"image {index}: {h}x{w} makes a {n}-byte stream, more than "
                         f"{MAX_STREAM}")
    return h, w


def _align(n, a):
    return -(-n // a) * a


class Plan:
    """One batch laid out for the device: desc (without the image addresses, which `set_sources`
    fills in) and the size of every device buffer.  Sizes depend on the shapes only."""

    def __init__(self, images_meta):
        """images_meta: one (shape, dtype) per image."""
        self.B = B = len(images_meta)
        desc = np.zeros((B, DESC_WORDS), dtype=np.int64)
        stream = tiles = stretch = blocks = blkpos = zbuf = out = 0
        self.max_n = self.max_blocks = self.max_chunks = 1
        self.shapes = []
        for b, (shape, dtype) in enumerate(images_meta):
            h, w = check_image(shape, dtype, b)
            self.shapes.append((h, w))
            n = stream_length(h, w)
            nt = -(-n // TILE)
            cap = n // 2 + 1
            mb = max_blocks(n)
            zwords = _align(deflate_bound(n), 16) // 4
            chunks = -(-zlib_bound(n) // IDAT_BYTES)
            D = desc[b]
            D[D_H], D[D_W], D[D_N] = h, w, n
            D[D_STREAM_OFF], D[D_TILE_OFF], D[D_NTILES] = stream, tiles, nt
            D[D_STRETCH_OFF], D[D_STRETCH_CAP] = stretch, cap
            D[D_BLK_OFF], D[D_MAXBLK], D[D_BLKPOS_OFF] = blocks, mb, blkpos
            D[D_ZBUF_OFF], D[D_OUT_OFF] = zbuf, out
            D[D_WBITS] = window_bits(n)[1]
            D[D_CMF], D[D_FLG] = zlib_header(n)
            stream += _align(n, 16)
            tiles += nt
            stretch += 2 * cap
            blocks += mb
            blkpos += mb + 1
            zbuf += zwords
            out += _align(png_bound(n), 16)
            self.max_n = max(self.max_n, n)
            self.max_blocks = max(self.max_blocks, mb)
            self.max_chunks = max(self.max_chunks, chunks)
        self.desc = desc
        self.stream_bytes = max(stream, 16)
        self.total_tiles = tiles
        self.stretch_words = max(stretch, 1)
        self.blocks = max(blocks, 1)
        self.blkpos_words = max(blkpos, 1)
        self.zbuf_words = max(zbuf, 4)
        self.out_bytes = max(out, 16)

    def set_sources(self, addresses):
        """The device address of each image's contiguous H x W x 3 bytes."""
        self.desc[:, D_SRC] = np.asarray(addresses, dtype=np.int64)


# ---------------------------------------------------------------------------------- decoding
SIGNATURE = b"\x89PNG\r\n\x1a\n"
MAX_DIM = 1000000                 # libpng's default user width and height limit
MAX_DECODE_PIXELS = 1 << 30       # cv2's CV_IO_MAX_IMAGE_PIXELS
MAX_FILE_BYTES = 1 << 27          # mrx.h MRX_PNG_DEC_MAX_FILE: bit positions stay in int32
MAX_FILTERED = 1 << 30            # mrx.h MRX_PNG_DEC_MAX_FILTERED
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
ADAM7 = ((0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2),
         (0, 1, 1, 2))                                 # (x0, y0, dx, dy) of the seven passes
_APNG = (b"acTL", b"fcTL", b"fdAT")

# ---- the decoder's descriptor: int64 words per image (csrc/png_decode.cu, DD_*) ----
(DD_Z_OFF, DD_Z_LEN, DD_FILT_OFF, DD_N, DD_H, DD_W, DD_CT, DD_DEPTH, DD_INTERLACE, DD_ORIENT,
 DD_PLTE_N, DD_BLK_OFF, DD_BLK_CAP, DD_WSIZE, DD_TILE_OFF, DD_NTILES) = range(16)
DD_WORDS = 16
CK_IMG, CK_SRC, CK_LEN, CK_DST = range(4)            # int64 words per IDAT chunk
CK_WORDS = 4
DEC_INFO_WORDS = 8                                   # mrx.h MRX_PNG_DEC_INFO_WORDS
TILE_BITS = 1024                                     # mrx.h MRX_PNG_DEC_TILE_BITS
DEFAULT_SLOTS = 4                                    # candidate block starts kept per tile


class PngError(ValueError):
    """A file the device decoder does not accept (or whose image data is corrupt)."""


class DecodeHeader:
    """What `parse` found: geometry, colour type and depth, the palette, the IDAT chunks, the
    zlib window and the orientation."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    @property
    def shape(self):
        """(H, W, 3) of the decoded, oriented image."""
        if self.orientation >= 5:
            return (self.width, self.height, 3)
        return (self.height, self.width, 3)


def passes(h, w, interlace):
    """(width, height) of every non-empty pass: the image, or its Adam7 passes in order."""
    if not interlace:
        return [(w, h)]
    out = []
    for x0, y0, dx, dy in ADAM7:
        pw, ph = max(0, -(-(w - x0) // dx)), max(0, -(-(h - y0) // dy))
        if pw and ph:
            out.append((pw, ph))
    return out


def filtered_length(h, w, ct, depth, interlace):
    """Bytes of the filtered stream: per pass, per row a filter byte and the packed samples."""
    bits = CHANNELS[ct] * depth
    return sum(ph * (1 + (pw * bits + 7) // 8) for pw, ph in passes(h, w, interlace))


def _critical(tag):
    return not tag[0] & 0x20


def parse(blob, index=0):
    """Walk the chunks of one PNG file.  Returns a DecodeHeader; raises PngError.

    Refused, as libpng refuses them: a bad signature, IHDR or chunk layout, a CRC error on a
    critical chunk, an unknown critical chunk, a colour type / bit depth pair PNG does not define,
    a missing PLTE for colour type 3, IDAT chunks that are not consecutive, no IEND, a size past
    libpng's 1 000 000 limit or cv2's 2^30 pixels, a zlib header with CM != 8, CINFO > 7, FDICT
    set or a bad FCHECK; an empty PLTE in an RGB file, a PLTE of a palette file whose length is
    not 3 to 768 and a multiple of 3.  Refused besides, though libpng reads them: APNG (acTL,
    fcTL, fdAT), a repeated PLTE or one after IDAT, and a file or filtered stream larger than the
    device limits.  Ignored, as libpng ignores them: ancillary chunks (one whose CRC is wrong is
    discarded, an eXIf too; of two eXIf chunks the first counts), PLTE in a gray file and any
    non-empty one in an RGB file, bytes after IEND."""
    data = bytes(blob)

    def fail(reason):
        raise PngError(f"image {index}: {reason}")

    if data[:8] != SIGNATURE:
        fail("not a PNG file (bad signature)")
    if len(data) > MAX_FILE_BYTES:
        fail(f"file of {len(data)} bytes is larger than {MAX_FILE_BYTES}")
    p, ihdr, plte, idat, orient, seen_exif, ended = 8, None, None, [], 1, False, False
    idat_closed = False
    while not ended:
        if p + 12 > len(data):
            fail("truncated file (no IEND chunk)")
        n = struct.unpack(">I", data[p:p + 4])[0]
        tag = data[p + 4:p + 8]
        if n > 0x7FFFFFFF or p + 12 + n > len(data):
            fail(f"truncated {tag!r} chunk")
        if not all(65 <= c <= 90 or 97 <= c <= 122 for c in tag):
            fail(f"invalid chunk type {tag!r}")
        body = data[p + 8:p + 8 + n]
        crc_ok = zlib.crc32(tag + body) == struct.unpack(">I", data[p + 8 + n:p + 12 + n])[0]
        name = tag.decode("ascii")
        if ihdr is None and tag != b"IHDR":
            fail("the first chunk is not IHDR")
        if tag in _APNG:
            fail(f"APNG ({name} chunk): animated PNG files are not supported")
        if _critical(tag) and tag != b"IDAT" and not crc_ok:
            fail(f"{name}: CRC error")
        if idat and tag != b"IDAT":
            idat_closed = True
        if tag == b"IHDR":
            if ihdr is not None:
                fail("two IHDR chunks")
            if n != 13:
                fail("bad IHDR length")
            ihdr = struct.unpack(">IIBBBBB", body)
        elif tag == b"PLTE":
            if plte is not None or idat:
                fail("PLTE repeated or after IDAT (not decoded on the device)")
            plte = body
        elif tag == b"IDAT":
            if idat_closed:
                fail("IDAT chunks are not consecutive")
            idat.append((p + 4, n))
        elif tag == b"IEND":
            ended = True
        elif _critical(tag):
            fail(f"unknown critical chunk {name}")
        elif tag == b"eXIf" and crc_ok and not seen_exif:      # the first one counts
            orient, seen_exif = exif.orientation(body), True
        p += 12 + n
    w, h, depth, ct, comp, filt, interlace = ihdr
    if w == 0 or h == 0 or w > MAX_DIM or h > MAX_DIM:
        fail(f"image size {w}x{h} outside [1, {MAX_DIM}]")
    if ct not in DEPTHS or depth not in DEPTHS[ct]:
        fail(f"invalid colour type {ct} with bit depth {depth}")
    if comp != 0 or filt != 0 or interlace > 1:
        fail("unknown compression, filter or interlace method")
    if w * h > MAX_DECODE_PIXELS:
        fail(f"{h}x{w} is more than {MAX_DECODE_PIXELS} pixels (cv2.imdecode refuses it too)")
    if ct == 3 and plte is None:
        fail("missing PLTE for a palette image")
    # libpng ignores PLTE in a gray file; in an RGB file it ignores any but an empty one
    if ct == 3 and (len(plte) == 0 or len(plte) % 3 or len(plte) > 768):
        fail(f"invalid PLTE length {len(plte)}")
    if ct in (2, 6) and plte is not None and len(plte) == 0:
        fail("invalid PLTE length 0")
    if not idat:
        fail("no IDAT chunk")
    nfilt = filtered_length(h, w, ct, depth, interlace)
    if nfilt > MAX_FILTERED:
        fail(f"{nfilt} filtered bytes, more than {MAX_FILTERED}")
    head = b"".join(data[s + 4:s + 4 + k] for s, k in idat[:3])[:2]
    if len(head) < 2:
        fail("truncated zlib stream (Not enough image data)")
    cmf, flg = head[0], head[1]
    if cmf & 15 != 8:
        fail("zlib: unknown compression method")
    if cmf >> 4 > 7:
        fail("zlib: invalid window size")
    if (cmf * 256 + flg) % 31:
        fail("zlib: incorrect header check")
    if flg & 32:
        fail("zlib: missing LZ dictionary")
    pal = np.zeros((256, 3), np.uint8)
    npal = 0
    if ct == 3:
        npal = len(plte) // 3
        pal[:npal] = np.frombuffer(plte, np.uint8).reshape(-1, 3)
    return DecodeHeader(width=w, height=h, color_type=ct, depth=depth, interlace=interlace,
                        palette=pal, palette_len=npal, orientation=orient, idat=idat,
                        zlib_len=sum(k for _, k in idat), window=1 << ((cmf >> 4) + 8),
                        filtered=nfilt, file_len=len(data))


def block_capacity(filtered, zlib_len):
    """Deflate blocks listed per image: every block takes at least 10 bits of the stream; at
    most one per 64 filtered bytes is listed (an image with more is expanded by one warp)."""
    return min(8 * zlib_len // 10 + 1, filtered // 64 + 64)


class DecodePlan:
    """One batch of PNG files laid out for `mrx_png_decode`: the upload (files, desc, chunks,
    palettes) and the size of every device buffer.  Sizes depend on the headers and the file
    lengths only.  index[b]: the caller's index of file b, named in refusals.  slots: candidate
    block starts kept per tile of TILE_BITS stream bits (0: the chain measures every block)."""

    def __init__(self, blobs, index=None, slots=DEFAULT_SLOTS):
        if not 0 <= slots <= 32:
            raise ValueError(f"slots={slots} outside [0, 32]")
        self.K = int(slots)
        from .jpeg import _as_bytes

        index = list(range(len(blobs))) if index is None else list(index)
        datas = [_as_bytes(b, i) for i, b in zip(index, blobs)]
        self.headers = [parse(d, i) for i, d in zip(index, datas)]
        self.B = B = len(datas)
        desc = np.zeros((B, DD_WORDS), dtype=np.int64)
        chunks = []
        plte = np.zeros((B, 768), dtype=np.uint8)
        file_off = z = filt = blk = tiles = 0
        self.max_n = self.max_zlen = 2
        self.max_pixels = self.max_tiles = self.max_blocks = 1
        for b, hd in enumerate(self.headers):
            D = desc[b]
            D[DD_Z_OFF], D[DD_Z_LEN], D[DD_FILT_OFF], D[DD_N] = z, hd.zlib_len, filt, hd.filtered
            D[DD_H], D[DD_W], D[DD_CT], D[DD_DEPTH] = hd.height, hd.width, hd.color_type, hd.depth
            D[DD_INTERLACE], D[DD_ORIENT], D[DD_PLTE_N] = hd.interlace, hd.orientation, \
                hd.palette_len
            cap = block_capacity(hd.filtered, hd.zlib_len)
            D[DD_BLK_OFF], D[DD_BLK_CAP], D[DD_WSIZE] = blk, cap, hd.window
            nt = -(-8 * hd.zlib_len // TILE_BITS)
            D[DD_TILE_OFF], D[DD_NTILES] = tiles, nt
            dst = 0
            for s, k in hd.idat:
                chunks.append((b, file_off + s, k, dst))
                dst += k
            plte[b] = hd.palette.reshape(-1)
            file_off += _align(hd.file_len, 16)
            z += _align(hd.zlib_len, 16)
            filt += _align(hd.filtered, 16)
            blk += cap
            tiles += nt
            self.max_n = max(self.max_n, hd.filtered)
            self.max_zlen = max(self.max_zlen, hd.zlib_len)
            self.max_tiles = max(self.max_tiles, nt)
            self.max_blocks = max(self.max_blocks, cap)
            self.max_pixels = max(self.max_pixels, hd.height * hd.width)
        files = np.zeros(max(file_off, 16), dtype=np.uint8)
        o = 0
        for d, hd in zip(datas, self.headers):
            files[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
            o += _align(hd.file_len, 16)
        self.files, self.desc, self.plte = files, desc, plte
        self.chunks = np.asarray(chunks or [(0, 0, 0, 0)], dtype=np.int64).reshape(-1, CK_WORDS)
        self.n_chunks = len(chunks)
        self.z_bytes = max(z, 16)
        self.filt_bytes = max(filt, 16)
        self.total_tiles = max(tiles, 1)
        self.block_words = 2 * max(blk, 1)
        self.shapes = [hd.shape for hd in self.headers]


def status_reasons(bits):
    """Reasons for a nonzero device status word (mrx.h MRX_PNG_ST_*), in libpng's words."""
    names = [(1, "IDAT: CRC error"), (2, "Not enough image data"),
             (4, "invalid block type, code lengths, code or stored block length"),
             (8, "invalid distance too far back"), (16, "incorrect data check (Adler-32)"),
             (32, "bad adaptive filter value")]
    return ", ".join(n for bit, n in names if bits & bit)
