"""Host half of the device PNG encoder (csrc/png.cu, `mrx_png_encode`).

NumPy only.  `Plan` checks each image and lays the batch out from the images' sizes alone: the
filtered stream length n = H * (3W + 1), the window bits cv2 writes into the zlib header, every
device buffer's offsets and a worst-case bound on each file, so that every buffer is sized before
anything runs.  What is encoded is what `cv2.imwrite(path, rgb[..., ::-1])` writes for a uint8
H x W x 3 RGB image (tests/png_oracle.py states how); anything else raises ValueError naming the
image's index.
"""
from __future__ import annotations

import numpy as np

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
