"""NumPy restatement of the baseline JPEG file cv2.imencode('.jpg', rgb[..., ::-1], [quality,
optimize]) writes (libjpeg-turbo's jcapistd/jcmarker/jccolor/jcsample/jcprepct/jfdctint/jcdctmgr/
jccoefct/jchuff), the definition csrc/jpeg_encode.cu is tested against.

`encode(img, quality, optimize)` returns (file bytes, Encoded): the quantised coefficients of every
block of the scan in MCU order (zigzag, dummy blocks included), the coded bit count, the unstuffed
byte count, the stuffed 0x00 count and the header length.  Integer arithmetic throughout, in int64.
"""
from __future__ import annotations

import struct
from types import SimpleNamespace

import numpy as np

from jpeg_reencode import _optimal_table
from matterport_maskrcnn_with_tensorflow_serving_b200.jpeg import ZIGZAG as _ZZ

ZIGZAG = _ZZ[:64]

# T.81 Annex K.1 (natural order)
STD_QUANT = np.array([
    [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69,
     56, 14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81,
     104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99],
    [17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99,
     99, 47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32], dtype=np.int64)

# T.81 Annex K.3: (bits[16], vals) of DC luma, AC luma, DC chroma, AC chroma
_AC_LUMA_VALS = bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25"
    "262728292a3435363738393a434445464748494a535455565758595a636465666768696a737475767778797a83"
    "8485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3"
    "d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa")
_AC_CHROMA_VALS = bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f1171819"
    "1a262728292a35363738393a434445464748494a535455565758595a636465666768696a737475767778797a8283"
    "8485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4"
    "d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa")
STD_TABLES = [
    ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12))),
    ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], list(_AC_LUMA_VALS)),
    ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12))),
    ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], list(_AC_CHROMA_VALS)),
]


def quant_tables(quality):
    """jpeg_set_quality(quality, force_baseline=TRUE): [2, 64] natural order."""
    q = max(1, min(int(quality), 100))
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((STD_QUANT * scale + 50) // 100, 1, 255)


def ycc(img):
    """jccolor.c rgb_ycc_convert: int64 Y, Cb, Cr planes of a uint8 RGB image."""
    r, g, b = (img[..., i].astype(np.int64) for i in range(3))
    half, off = 1 << 15, (128 << 16) + (1 << 15) - 1
    y = (19595 * r + 38470 * g + 7471 * b + half) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + off) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + off) >> 16
    return y, cb, cr


def geometry(h, w):
    """(MCU columns, MCU rows, luma blocks across, luma blocks down)."""
    return -(-w // 16), -(-h // 16), -(-w // 8), -(-h // 8)


def planes(img):
    """The sample planes the FDCT reads: luma [16 * mcuy, 8 * wib] and the two chroma planes
    [8 * mcuy, 8 * mcux], with the edge replication and h2v2 downsampling of jcprepct/jcsample."""
    h, w = img.shape[:2]
    mcux, mcuy, wib, hib = geometry(h, w)
    y, cb, cr = ycc(img)
    rows = np.minimum(np.arange(16 * mcuy), h - 1)
    luma = y[rows][:, np.minimum(np.arange(8 * wib), w - 1)]
    ch = []
    for p in (cb, cr):
        full = p[np.minimum(np.arange(2 * (-(-h // 2))), h - 1)]
        full = full[:, np.minimum(np.arange(16 * mcux), w - 1)]
        s = full[0::2, 0::2] + full[0::2, 1::2] + full[1::2, 0::2] + full[1::2, 1::2]
        bias = 1 + (np.arange(s.shape[1]) & 1)
        d = (s + bias) >> 2
        ch.append(d[np.minimum(np.arange(8 * mcuy), d.shape[0] - 1)])
    return luma, ch[0], ch[1]


def fdct_islow(blocks):
    """jfdctint.c on int64 [n, 8, 8] samples - 128 (CONST_BITS 13, PASS1_BITS 2)."""
    d = blocks.astype(np.int64).copy()

    def one_pass(d, first):
        x = [d[..., i] for i in range(8)]
        t0, t7 = x[0] + x[7], x[0] - x[7]
        t1, t6 = x[1] + x[6], x[1] - x[6]
        t2, t5 = x[2] + x[5], x[2] - x[5]
        t3, t4 = x[3] + x[4], x[3] - x[4]
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        sh = 11 if first else 15

        def desc(v, n):
            return (v + (1 << (n - 1))) >> n

        out = [None] * 8
        if first:
            out[0], out[4] = (t10 + t11) << 2, (t10 - t11) << 2
        else:
            out[0], out[4] = desc(t10 + t11, 2), desc(t10 - t11, 2)
        z1 = (t12 + t13) * 4433
        out[2] = desc(z1 + t13 * 6270, sh)
        out[6] = desc(z1 - t12 * 15137, sh)
        z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
        z5 = (z3 + z4) * 9633
        a4, a5, a6, a7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
        z1, z2 = z1 * -7373, z2 * -20995
        z3, z4 = z3 * -16069 + z5, z4 * -3196 + z5
        out[7] = desc(a4 + z1 + z3, sh)
        out[5] = desc(a5 + z2 + z4, sh)
        out[3] = desc(a6 + z2 + z3, sh)
        out[1] = desc(a7 + z1 + z4, sh)
        return np.stack(out, axis=-1)

    d = one_pass(d, True)                                   # rows
    d = one_pass(d.transpose(0, 2, 1), False).transpose(0, 2, 1)   # columns
    return d


def quantize(c, q):
    """c / (8q), rounded half away from zero (jcdctmgr.c)."""
    d = 8 * q
    return np.sign(c) * ((np.abs(c) + d // 2) // d)


def _blocks(plane):
    return plane.reshape(plane.shape[0] // 8, 8, plane.shape[1] // 8, 8).transpose(0, 2, 1, 3)


def coefficients(img, quality=95):
    """int64 [6 * MCUs, 64]: the quantised zigzag coefficients of every block of the scan in MCU
    order (Y00 Y01 Y10 Y11 Cb Cr), dummy blocks included (jccoefct.c)."""
    h, w = img.shape[:2]
    mcux, mcuy, wib, hib = geometry(h, w)
    qt = quant_tables(quality)
    luma, cb, cr = planes(img)
    out = np.zeros((mcuy, mcux, 6, 64), np.int64)
    lb = _blocks(luma - 128)                 # [2 * mcuy, wib, 8, 8]
    lq = quantize(fdct_islow(lb.reshape(-1, 8, 8)).reshape(-1, 64), qt[0])
    lq = lq.reshape(2 * mcuy, wib, 64)[:hib]
    grid = np.zeros((2 * mcuy, 2 * mcux, 64), np.int64)
    grid[:hib, :wib] = lq
    if wib % 2:                                     # right dummy column: the DC on its left
        grid[:hib, wib, 0] = grid[:hib, wib - 1, 0]
    if hib % 2:                                     # dummy row: the MCU's last block above
        grid[hib, :, 0] = np.repeat(grid[hib - 1, 1::2, 0], 2)
    out[:, :, :4] = grid.reshape(mcuy, 2, mcux, 2, 64).transpose(0, 2, 1, 3, 4).reshape(
        mcuy, mcux, 4, 64)
    for ci, p in ((4, cb), (5, cr)):
        cbk = _blocks(p - 128).reshape(-1, 8, 8)
        out[:, :, ci] = quantize(fdct_islow(cbk).reshape(-1, 64), qt[1]).reshape(mcuy, mcux, 64)
    return out.reshape(-1, 64)[:, ZIGZAG]


def _nbits(v):
    a = np.abs(v)
    n = np.zeros(a.shape, np.int64)
    while (a > 0).any():
        n += a > 0
        a = a >> 1
    return n


def symbols(coef):
    """Every symbol of the scan in order: (table 0..3, symbol, value bits, value length) as int64
    arrays (jchuff.c encode_one_block; DC predicted per component in MCU order)."""
    nb = coef.shape[0]
    comp = np.tile(np.array([0, 0, 0, 0, 1, 2]), nb // 6)
    dc = coef[:, 0]
    pred = np.zeros(nb, np.int64)
    for c in range(3):
        idx = np.nonzero(comp == c)[0]
        pred[idx[1:]] = dc[idx[:-1]]
    tdc = np.where(comp == 0, 0, 2)
    diff = dc - pred
    # events keyed by (block, position, order): DC at position 0, ZRLs and the coefficient at
    # its position, EOB at 64
    ev = [[], [], [], [], []]                      # keys, tables, symbols, values, lengths

    def add(blk, pos, sub, *fields):
        key = (np.asarray(blk, np.int64) * 65 + pos) * 4 + sub
        for lst, x in zip(ev, (key,) + fields):
            lst.append(np.broadcast_to(np.asarray(x, np.int64), key.shape))

    n = _nbits(diff)
    add(np.arange(nb), 0, 0, tdc, n, np.where(diff < 0, diff - 1, diff) & ((1 << n) - 1), n)
    ac = coef[:, 1:]
    b, z = np.nonzero(ac)
    pos = z + 1
    prev = np.zeros(len(pos), np.int64)
    same = b[1:] == b[:-1]                       # the previous nonzero is in the same block
    prev[1:][same] = pos[:-1][same]
    run = pos - prev - 1
    zrl = run // 16
    r = run % 16
    v = ac[b, z]
    m = _nbits(v)
    for k in range(1, 4):                           # at most 3 ZRLs before a coefficient
        sel = zrl >= k
        add(b[sel], pos[sel], k - 1, tdc[b[sel]] + 1, np.full(sel.sum(), 0xF0), 0, 0)
    add(b, pos, 3, tdc[b] + 1, (r << 4) + m, np.where(v < 0, v - 1, v) & ((1 << m) - 1), m)
    last = np.zeros(nb, np.int64)
    np.maximum.at(last, b, pos)
    eob = np.nonzero(last < 63)[0]
    add(eob, 64, 0, tdc[eob] + 1, np.zeros(len(eob), np.int64), 0, 0)
    keys, tabs, syms, vals, lens = (np.concatenate(x) for x in ev)
    order = np.argsort(keys, kind="stable")
    return tabs[order], syms[order], vals[order], lens[order]


def code_table(bits, vals):
    """(code, length) per symbol [256] (jpeg_make_c_derived_tbl)."""
    code = np.zeros(256, np.int64)
    size = np.zeros(256, np.int64)
    c, k = 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            code[vals[k]], size[vals[k]] = c, ln
            c += 1
            k += 1
        c <<= 1
    return code, size


def _pack(values, lengths):
    """The bits of (value, length) pairs, most significant first, 1-padded to a byte."""
    total = int(lengths.sum())
    ends = np.cumsum(lengths)
    owner = np.repeat(np.arange(len(lengths)), lengths)
    shift = ends[owner] - 1 - np.arange(total)
    bits = ((values[owner] >> shift) & 1).astype(np.uint8)
    pad = (-total) % 8
    bits = np.concatenate([bits, np.ones(pad, np.uint8)])
    return np.packbits(bits).tobytes(), total


def _segment(code, payload):
    return b"\xff" + bytes([code]) + struct.pack(">H", len(payload) + 2) + payload


def encode(img, quality=95, optimize=False):
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape[:2]
    coef = coefficients(img, quality)
    tab, sym, val, ln = symbols(coef)
    if optimize:
        tables = []
        for t in range(4):
            freq = np.bincount(sym[tab == t], minlength=256)
            bits, vals = _optimal_table([int(f) for f in freq])
            tables.append((list(bits), list(vals)))
    else:
        tables = STD_TABLES
    codes = [code_table(*t) for t in tables]
    code = np.zeros(len(sym), np.int64)
    size = np.zeros(len(sym), np.int64)
    for t in range(4):
        s = tab == t
        code[s], size[s] = codes[t][0][sym[s]], codes[t][1][sym[s]]
    vals = np.stack([code, val], 1).ravel()
    lens = np.stack([size, ln], 1).ravel()
    data, nbits = _pack(vals, lens)
    arr = np.frombuffer(data, np.uint8)
    ff = np.nonzero(arr == 0xFF)[0]
    stuffed = np.insert(arr, ff + 1, 0).tobytes()
    qt = quant_tables(quality)
    head = b"\xff\xd8" + _segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t in range(2):
        head += _segment(0xDB, bytes([t]) + bytes(qt[t][ZIGZAG].astype(np.uint8)))
    head += _segment(0xC0, struct.pack(">BHHB", 8, h, w, 3) + bytes([1, 0x22, 0, 2, 0x11, 1, 3,
                                                                      0x11, 1]))
    for t, (bits, vs) in enumerate(tables):
        head += _segment(0xC4, bytes([((t & 1) << 4) | (t >> 1)]) + bytes(bits) + bytes(vs))
    head += _segment(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))
    out = head + stuffed + b"\xff\xd9"
    return out, SimpleNamespace(coef=coef, bits=nbits, bytes=len(data), ff=len(ff),
                                hdr=len(head), tables=tables)
