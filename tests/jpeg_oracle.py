"""CPU restatement of libjpeg-turbo's baseline decode path as cv2.imdecode(IMREAD_COLOR) runs it
(JDCT_ISLOW, fancy upsampling), loop for loop, for the device decoder's tests.

Held bit for bit to cv2.imdecode by tests/test_jpeg_oracle.py, so it is pinned to the real library.
The marker walk is the package's `jpeg.parse` (whose refusals test_host_jpeg.py covers); everything
after it is restated here: jdhuff.c's decode_mcu (with the 16 guard entries of the natural-order
table), the restart handling, jidctint.c's jpeg_idct_islow with the post-IDCT range-limit table,
jdsample.c's upsamplers with the context rows of jdmainct.c, jdcolor.c's ycc_rgb_convert and
OpenCV's EXIF orientation.  Corrupt entropy-coded data raises JpegError (libjpeg-turbo warns and
substitutes zeros: a stated difference of the device decoder, which refuses the same files).
"""
from __future__ import annotations

import numpy as np

from matterport_maskrcnn_with_tensorflow_serving_b200 import jpeg as J

CONST_BITS, PASS1_BITS = 13, 2
FIX_0_298631336, FIX_0_390180644, FIX_0_541196100 = 2446, 3196, 4433
FIX_0_765366865, FIX_0_899976223, FIX_1_175875602 = 6270, 7373, 9633
FIX_1_501321110, FIX_1_847759065, FIX_1_961570560 = 12299, 15137, 16069
FIX_2_053119869, FIX_2_562915447, FIX_3_072711026 = 16819, 20995, 25172


class _Bits:
    """jdhuff.c's bit source over the entropy-coded bytes: 0xFF00 is 0xFF, a marker ends the data
    (reading on past it is corrupt data here), RSTn is consumed by `restart`."""

    def __init__(self, data, pos):
        self.data, self.pos = data, pos
        self.acc, self.n = 0, 0
        self.marker = None

    def _fill(self):
        d = self.data
        if self.marker is None and self.pos < len(d):
            c = d[self.pos]
            if c == 0xFF:
                nxt = d[self.pos + 1] if self.pos + 1 < len(d) else 0xD9
                if nxt == 0x00:
                    self.pos += 2
                else:
                    self.marker = nxt
                    raise J.JpegError("data ended before the last MCU")
            else:
                self.pos += 1
            self.acc = (self.acc << 8) | c
            self.n += 8
            return
        raise J.JpegError("data ended before the last MCU")

    def bit(self):
        if self.n == 0:
            self._fill()
        self.n -= 1
        return (self.acc >> self.n) & 1

    def bits(self, s):
        v = 0
        for _ in range(s):
            v = (v << 1) | self.bit()
        return v

    def restart(self, k):
        self.acc, self.n = 0, 0
        d = self.data
        if self.marker is None:
            if self.pos + 1 >= len(d) or d[self.pos] != 0xFF:
                raise J.JpegError("missing or out-of-order RST marker")
            self.marker = d[self.pos + 1]
            self.pos += 2
        else:
            self.pos += 2
        if self.marker != 0xD0 + (k & 7):
            raise J.JpegError("missing or out-of-order RST marker")
        self.marker = None


def _huff(bits, t):
    """jpeg_huff_decode: canonical codes one bit at a time."""
    code = bits.bit()
    length = 1
    while length <= 16 and (t.maxcode[length] < 0 or code > t.maxcode[length]):
        code = (code << 1) | bits.bit()
        length += 1
    if length > 16:
        raise J.JpegError("bad Huffman code")
    return t.vals[t.valptr[length] + code]


def _extend(r, s):
    return r - (1 << s) + 1 if r < (1 << (s - 1)) else r


def coefficients(blob):
    """Quantised coefficients in decode order: int16 [MCUs * blocks_per_mcu, 64], natural order,
    DC after the prediction (JCOEF), plus the parsed header."""
    data = bytes(blob)
    hd = J.parse(data)
    mcus = hd.mcux * hd.mcuy
    ri = hd.restart_interval or mcus
    comp_of = [ci for ci, (h, v) in enumerate(hd.samp) for _ in range(h * v)]
    out = np.zeros((mcus * hd.bpm, 64), dtype=np.int16)
    bits = _Bits(data, hd.scan_off)
    last_dc = [0] * hd.ncomp
    blk = 0
    for m in range(mcus):
        if m and m % ri == 0:
            bits.restart(m // ri - 1)
            last_dc = [0] * hd.ncomp
        for c in range(hd.bpm):
            ci = comp_of[c]
            dct, act, _ = hd.tables[ci]
            s = _huff(bits, dct)
            diff = _extend(bits.bits(s), s) if s else 0
            dcv = last_dc[ci] + diff
            if not -2 ** 31 <= dcv < 2 ** 31:
                raise J.JpegError("DC coefficient overflows int32")
            last_dc[ci] = dcv
            blockv = [0] * 64
            blockv[0] = ((dcv + 32768) & 0xFFFF) - 32768
            k = 1
            while k < 64:
                rs = _huff(bits, act)
                r, s = rs >> 4, rs & 15
                if s:
                    k += r
                    v = _extend(bits.bits(s), s)
                    blockv[J.ZIGZAG[k]] = v
                else:
                    if r != 15:
                        break
                    k += 15
                k += 1
            out[blk] = blockv
            blk += 1
    return out, hd


def _range_limit():
    """jdmaster.c prepare_range_limit_table, seen from IDCT_range_limit (index x & 1023)."""
    v = np.arange(1024)
    return np.where(v < 128, v + 128, np.where(v < 512, 255, np.where(v < 896, 0, v - 896))
                    ).astype(np.uint8)


def idct_islow(coef, quant):
    """jidctint.c jpeg_idct_islow over [N, 64] blocks -> uint8 [N, 8, 8] (vectorised, int64)."""
    x = coef.astype(np.int64).reshape(-1, 8, 8) * quant.astype(np.int64).reshape(1, 8, 8)

    def one_d(i0, i1, i2, i3, i4, i5, i6, i7):
        z2, z3 = i2, i6
        z1 = (z2 + z3) * FIX_0_541196100
        tmp2 = z1 + z3 * -FIX_1_847759065
        tmp3 = z1 + z2 * FIX_0_765366865
        tmp0 = (i0 + i4) << CONST_BITS
        tmp1 = (i0 - i4) << CONST_BITS
        t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
        t0, t1, t2, t3 = i7, i5, i3, i1
        z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
        z5 = (z3 + z4) * FIX_1_175875602
        t0, t1 = t0 * FIX_0_298631336, t1 * FIX_2_053119869
        t2, t3 = t2 * FIX_3_072711026, t3 * FIX_1_501321110
        z1, z2 = z1 * -FIX_0_899976223, z2 * -FIX_2_562915447
        z3, z4 = z3 * -FIX_1_961570560 + z5, z4 * -FIX_0_390180644 + z5
        t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
        return [t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3]

    def descale(v, n):
        return (v + (1 << (n - 1))) >> n

    # pass 1: columns (the all-zero-AC shortcut gives the same values)
    cols = one_d(*[x[:, k, :] for k in range(8)])
    ws = np.stack([descale(v, CONST_BITS - PASS1_BITS) for v in cols], axis=1)   # [N, 8, 8]
    rows = one_d(*[ws[:, :, k] for k in range(8)])
    out = np.stack([descale(v, CONST_BITS + PASS1_BITS + 3) for v in rows], axis=2)
    return _range_limit()[out & 1023]


def planes(blob):
    """IDCT output of every component at its full padded block size, plus the header."""
    coef, hd = coefficients(blob)
    res = []
    blk = coef.reshape(hd.mcuy, hd.mcux, hd.bpm, 64)
    c0 = 0
    for ci, (h, v) in enumerate(hd.samp):
        q = hd.tables[ci][2]
        sel = blk[:, :, c0:c0 + h * v].reshape(-1, 64)
        px = idct_islow(sel, q).reshape(hd.mcuy, hd.mcux, v, h, 8, 8)
        res.append(px.transpose(0, 2, 4, 1, 3, 5).reshape(hd.mcuy * v * 8, hd.mcux * h * 8))
        c0 += h * v
    return res, hd


def _upsample(p, he, ve, dw, dh, H, W):
    """jdsample.c: the method jinit_upsampler picks for (h_expand, v_expand), cropped to H x W."""
    p = p.astype(np.int32)
    if he == 1 and ve == 1:
        return p[:H, :W]
    fancy_h = dw > 2
    if he == 2 and ve == 1 and fancy_h:
        q = p[:, :dw]
        left = np.concatenate([q[:, :1], q[:, :-1]], axis=1)
        right = np.concatenate([q[:, 1:], q[:, -1:]], axis=1)
        even = (3 * q + left + 1) >> 2
        odd = (3 * q + right + 2) >> 2
        even[:, 0] = q[:, 0]
        odd[:, -1] = q[:, -1]
        out = np.stack([even, odd], axis=2).reshape(q.shape[0], 2 * dw)
        return out[:H, :W]
    if he == 1 and ve == 2:
        q = p[:dh, :]
        above = np.concatenate([q[:1], q[:-1]], axis=0)
        below = np.concatenate([q[1:], q[-1:]], axis=0)
        top = (3 * q + above + 1) >> 2
        bot = (3 * q + below + 2) >> 2
        out = np.stack([top, bot], axis=1).reshape(2 * dh, q.shape[1])
        return out[:H, :W]
    if he == 2 and ve == 2 and fancy_h:
        q = p[:dh, :dw]
        above = np.concatenate([q[:1], q[:-1]], axis=0)
        below = np.concatenate([q[1:], q[-1:]], axis=0)
        rows = []
        for nb in (above, below):
            cs = 3 * q + nb
            left = np.concatenate([cs[:, :1], cs[:, :-1]], axis=1)
            right = np.concatenate([cs[:, 1:], cs[:, -1:]], axis=1)
            even = (3 * cs + left + 8) >> 4
            odd = (3 * cs + right + 7) >> 4
            even[:, 0] = (4 * cs[:, 0] + 8) >> 4
            odd[:, -1] = (4 * cs[:, -1] + 7) >> 4
            rows.append(np.stack([even, odd], axis=2).reshape(dh, 2 * dw))
        out = np.stack(rows, axis=1).reshape(2 * dh, 2 * dw)
        return out[:H, :W]
    # int_upsample / h2v1_upsample / h2v2_upsample: replication
    return np.repeat(np.repeat(p, ve, axis=0), he, axis=1)[:H, :W]


def _ycc_rgb(y, cb, cr):
    """jdcolor.c ycc_rgb_convert with build_ycc_rgb_table's 16-bit fixed point."""
    def fix(x):
        return int(x * 65536 + 0.5)
    half = 1 << 15
    xcb, xcr = cb - 128, cr - 128
    r = y + ((fix(1.40200) * xcr + half) >> 16)
    g = y + ((-fix(0.71414) * xcr + (-fix(0.34414) * xcb + half)) >> 16)
    b = y + ((fix(1.77200) * xcb + half) >> 16)
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def orient(img, o):
    """OpenCV's ExifTransform for orientation o (1-8)."""
    if o == 2:
        return img[:, ::-1]
    if o == 3:
        return img[::-1, ::-1]
    if o == 4:
        return img[::-1]
    if o == 5:
        return img.transpose(1, 0, 2)
    if o == 6:
        return img.transpose(1, 0, 2)[:, ::-1]
    if o == 7:
        return img.transpose(1, 0, 2)[::-1, ::-1]
    if o == 8:
        return img.transpose(1, 0, 2)[::-1]
    return img


def decode(blob):
    """uint8 [H, W, 3] RGB: what cv2.cvtColor(cv2.imdecode(...), COLOR_BGR2RGB) returns."""
    pl, hd = planes(blob)
    H, W = hd.height, hd.width
    ups = []
    for ci, (h, v) in enumerate(hd.samp):
        dw = -(-W * h // hd.hmax)
        dh = -(-H * v // hd.vmax)
        ups.append(_upsample(pl[ci], hd.hmax // h, hd.vmax // v, dw, dh, H, W))
    if hd.color == J.COLOR_GRAY:
        img = np.repeat(ups[0][..., None], 3, axis=2).astype(np.uint8)
    elif hd.color == J.COLOR_RGB:
        img = np.stack(ups, axis=-1).astype(np.uint8)
    else:
        img = _ycc_rgb(*ups)
    return np.ascontiguousarray(orient(img, hd.orientation))
