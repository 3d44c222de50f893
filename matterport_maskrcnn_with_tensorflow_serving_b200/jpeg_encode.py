"""Host half of the device JPEG encoder (csrc/jpeg_encode.cu, `mrx_jpeg_encode`).

NumPy only.  `EncodePlan` checks each image and the quality and lays the batch out from the
images' sizes alone: the MCU grid, the scan's block count (six blocks per 16 x 16 MCU, dummy
blocks included), every device buffer's offsets and a worst-case bound on each file, so that every
buffer is sized before anything runs.  What is encoded is what
`cv2.imencode('.jpg', rgb[..., ::-1], [IMWRITE_JPEG_QUALITY, q, IMWRITE_JPEG_OPTIMIZE, opt])` writes
for a uint8 H x W x 3 RGB image (tests/jpeg_encode_oracle.py states how); anything else raises
ValueError naming the image's index.
"""
from __future__ import annotations

import numpy as np

BLOCK_TILE = 256                  # blocks per tile of the device's block passes
BYTE_TILE = 2048                  # entropy-coded bytes per tile of the stuffing passes
MAX_SIDE = 65535                  # mrx.h MRX_JPEG_ENC_MAX_SIDE: a baseline frame header's limit
TAB_BYTES = 16 + 256              # bits[16] and vals of one Huffman table
INFO_WORDS = 8                    # mrx.h MRX_JPEG_ENC_INFO_WORDS
# A block codes its DC (a code of at most 16 bits and at most 11 value bits) and at most 63 AC
# coefficients (at most 16 + 10 bits each; a ZRL or EOB only stands for zeros and costs less
# than the coefficients it replaces): 27 + 63 * 26 bits.
MAX_BLOCK_BITS = 27 + 63 * 26
# SOI, APP0, two DQT, SOF0, SOS and EOI, and four DHT holding at most 12 + 162 + 12 + 162 values
MAX_HEADER = 2 + 18 + 2 * 69 + 19 + 4 * 21 + 2 * (12 + 162) + 14

# ---- the device descriptor: int64 words per image (csrc/jpeg_encode.cu, D_*) ----
(D_SRC, D_H, D_W, D_MCUX, D_MCUY, D_NBLK, D_BLK_OFF, D_BT_OFF, D_NBT, D_WORD_OFF, D_YT_OFF,
 D_NYT, D_OUT_OFF) = range(13)
DESC_WORDS = 16


def blocks(h, w):
    """Blocks of the scan of an h x w image: four luma and two chroma per 16 x 16 MCU."""
    return 6 * (-(-h // 16)) * (-(-w // 16))


def data_bound(nblk):
    """Worst-case entropy-coded bytes of nblk blocks, before byte stuffing."""
    return -(-nblk * MAX_BLOCK_BITS // 8)


def file_bound(nblk):
    """Worst-case file bytes: the headers, every data byte stuffed, EOI."""
    return MAX_HEADER + 2 * data_bound(nblk) + 2


def check_quality(quality):
    """cv2's IMWRITE_JPEG_QUALITY range."""
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)):
        raise ValueError(f"quality {quality!r} is not an integer")
    if not 0 <= int(quality) <= 100:
        raise ValueError(f"quality {quality} outside [0, 100]")
    return int(quality)


def check_image(shape, dtype, index):
    """Refuse what the device encoder does not write as cv2.imencode('.jpg') would: anything but
    uint8 H x W x 3 with H, W in [1, 65535]."""
    if np.dtype(dtype) != np.uint8:
        raise ValueError(f"image {index}: dtype {np.dtype(dtype)} (expected uint8)")
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"image {index}: shape {tuple(shape)} (expected H x W x 3 RGB)")
    h, w = int(shape[0]), int(shape[1])
    if h == 0 or w == 0:
        raise ValueError(f"image {index}: {h}x{w} has no pixel")
    if h > MAX_SIDE or w > MAX_SIDE:
        raise ValueError(f"image {index}: {h}x{w} has a side over {MAX_SIDE}, more than a JPEG "
                         f"frame holds")
    return h, w


def _align(n, a):
    return -(-n // a) * a


class EncodePlan:
    """One batch laid out for the device: desc (without the image addresses, which `set_sources`
    fills in) and the size of every device buffer.  Sizes depend on the shapes only."""

    def __init__(self, images_meta, quality=95, optimize=False):
        """images_meta: one (shape, dtype) per image."""
        self.quality = check_quality(quality)
        self.optimize = bool(optimize)
        self.B = B = len(images_meta)
        desc = np.zeros((B, DESC_WORDS), dtype=np.int64)
        blk = btiles = words = ytiles = out = 0
        self.max_blocks = 6
        self.max_bytes = 1
        self.min_side, self.max_side = MAX_SIDE, 1
        self.shapes = []
        for b, (shape, dtype) in enumerate(images_meta):
            h, w = check_image(shape, dtype, b)
            self.shapes.append((h, w))
            nblk = blocks(h, w)
            nbt = -(-nblk // BLOCK_TILE)
            nbytes = data_bound(nblk)
            nyt = -(-nbytes // BYTE_TILE)
            D = desc[b]
            D[D_H], D[D_W] = h, w
            D[D_MCUX], D[D_MCUY], D[D_NBLK] = -(-w // 16), -(-h // 16), nblk
            D[D_BLK_OFF], D[D_BT_OFF], D[D_NBT] = blk, btiles, nbt
            D[D_WORD_OFF], D[D_YT_OFF], D[D_NYT], D[D_OUT_OFF] = words, ytiles, nyt, out
            blk += nblk
            btiles += nbt
            words += _align(nbytes + 4, 16) // 4
            ytiles += nyt
            out += _align(file_bound(nblk), 16)
            self.max_blocks = max(self.max_blocks, nblk)
            self.max_bytes = max(self.max_bytes, nbytes)
            self.min_side = min(self.min_side, h, w)
            self.max_side = max(self.max_side, h, w)
        self.desc = desc
        self.blocks = max(blk, 1)
        self.block_tiles = btiles
        self.byte_tiles = ytiles
        self.words = max(words, 4)
        self.out_bytes = max(out, 16)

    def set_sources(self, addresses):
        """The device address of each image's contiguous H x W x 3 bytes."""
        self.desc[:, D_SRC] = np.asarray(addresses, dtype=np.int64)
