"""CPU restatement of libjpeg-turbo's progressive Huffman decoder (jdphuff.c) as cv2.imdecode runs
it, loop for loop, for the device decoder's tests.

The marker walk and the scan-script checks are the package's `jpeg.parse_progressive`; everything
after it is restated here: the scan's block order (MCU order for an interleaved scan, the
component's own block grid for a single-component one), jdphuff.c's four decoders
(decode_mcu_DC_first, decode_mcu_AC_first, decode_mcu_DC_refine, decode_mcu_AC_refine) with the
EOB runs and process_restart.  The pixels then go through jpeg_oracle's IDCT, upsampling, colour and
orientation path, which the baseline oracle tests pin to cv2.  Corrupt entropy-coded data raises
JpegError, as the baseline oracle does.
"""
from __future__ import annotations

import numpy as np

import jpeg_oracle as JO
from matterport_maskrcnn_with_tensorflow_serving_b200 import jpeg as J


def scan_blocks(hd, sc):
    """Per MCU of the scan (an interleaved MCU, or one block of a single-component scan): the
    (component, coefficient row) of each of its blocks, rows in MCU decode order."""
    out = []
    if len(sc.comps) > 1:
        for m in range(sc.nmcu):
            blocks = []
            for ci, f in zip(sc.comps, sc.first):
                h, v = hd.samp[ci]
                blocks += [(ci, m * hd.bpm + f + dy * h + dx) for dy in range(v) for dx in range(h)]
            out.append(blocks)
        return out
    ci, f = sc.comps[0], sc.first[0]
    h, v = hd.samp[ci]
    for m in range(sc.nmcu):
        by, bx = divmod(m, sc.bw)
        out.append([(ci, ((by // v) * hd.mcux + bx // h) * hd.bpm + f + (by % v) * h + bx % h)])
    return out


def in_component_grid(hd):
    """bool [MCUs * blocks_per_mcu]: the blocks inside their component's own block grid.  A
    single-component scan codes only these; the MCU padding beyond them stays zero in a
    progressive file, where a baseline file codes it (the pixels there are cropped)."""
    out = np.zeros((hd.mcuy, hd.mcux, hd.bpm), dtype=bool)
    c0 = 0
    for h, v in hd.samp:
        bw = -(-(-(-hd.width * h // hd.hmax)) // 8)
        bh = -(-(-(-hd.height * v // hd.vmax)) // 8)
        for dy in range(v):
            for dx in range(h):
                ys = np.arange(hd.mcuy) * v + dy < bh
                xs = np.arange(hd.mcux) * h + dx < bw
                out[:, :, c0 + dy * h + dx] = ys[:, None] & xs[None, :]
        c0 += h * v
    return out.reshape(-1)


def _signed16(v):
    return ((v + 32768) & 0xFFFF) - 32768


def _decode_scan(data, hd, sc, coef):
    bits = JO._Bits(data, sc.data_off)
    nc = hd.ncomp
    p1 = 1 << sc.al
    m1 = -(1 << sc.al)
    last_dc, eobrun = [0] * nc, 0
    for m, blocks in enumerate(scan_blocks(hd, sc)):
        if m and m % sc.ri == 0:
            bits.restart(m // sc.ri - 1)
            last_dc, eobrun = [0] * nc, 0
        if sc.ss == 0 and sc.ah == 0:                        # decode_mcu_DC_first
            for i, (ci, row) in enumerate(blocks):
                t = sc.tables[sc.comps.index(ci)]
                s = JO._huff(bits, t)
                diff = JO._extend(bits.bits(s), s) if s else 0
                v = last_dc[ci] + diff
                if not -2 ** 31 <= v < 2 ** 31:
                    raise J.JpegError("DC coefficient overflows int32")
                last_dc[ci] = v
                coef[row, 0] = _signed16((v << sc.al) & 0xFFFFFFFF)
        elif sc.ss == 0:                                     # decode_mcu_DC_refine
            for ci, row in blocks:
                if bits.bit():
                    coef[row, 0] = _signed16(int(coef[row, 0]) | p1)
        elif sc.ah == 0:                                     # decode_mcu_AC_first
            (ci, row), = blocks
            if eobrun > 0:
                eobrun -= 1
                continue
            t = sc.tables[0]
            k = sc.ss
            while k <= sc.se:
                rs = JO._huff(bits, t)
                r, s = rs >> 4, rs & 15
                if s:
                    k += r
                    v = JO._extend(bits.bits(s), s)
                    coef[row, J.ZIGZAG[k]] = _signed16((v << sc.al) & 0xFFFFFFFF)
                elif r == 15:
                    k += 15
                else:
                    eobrun = 1 << r
                    if r:
                        eobrun += bits.bits(r)
                    eobrun -= 1
                    break
                k += 1
        else:                                                # decode_mcu_AC_refine
            (ci, row), = blocks
            blk = coef[row]
            t = sc.tables[0]
            k = sc.ss

            def correct(pos):
                if bits.bit() and (int(blk[pos]) & p1) == 0:
                    blk[pos] = _signed16(int(blk[pos]) + (p1 if blk[pos] >= 0 else m1))

            if eobrun == 0:
                while k <= sc.se:
                    rs = JO._huff(bits, t)
                    r, s = rs >> 4, rs & 15
                    if s:
                        s = p1 if bits.bit() else m1
                    elif r != 15:
                        eobrun = 1 << r
                        if r:
                            eobrun += bits.bits(r)
                        break
                    while k <= sc.se:
                        pos = J.ZIGZAG[k]
                        if blk[pos] != 0:
                            correct(pos)
                        else:
                            r -= 1
                            if r < 0:
                                break
                        k += 1
                    if s:
                        blk[J.ZIGZAG[k]] = s
                    k += 1
            if eobrun > 0:
                while k <= sc.se:
                    pos = J.ZIGZAG[k]
                    if blk[pos] != 0:
                        correct(pos)
                    k += 1
                eobrun -= 1


def coefficients(blob):
    """Quantised coefficients of a progressive file in MCU decode order (the layout of the
    baseline oracle and of the device), int16 [MCUs * blocks_per_mcu, 64], plus the header."""
    data = bytes(blob)
    hd, scans = J.parse_progressive(data)
    coef = np.zeros((hd.mcux * hd.mcuy * hd.bpm, 64), dtype=np.int16)
    for sc in scans:
        _decode_scan(data, hd, sc, coef)
    return coef, hd


def decode(blob, mistake=None):
    """uint8 [H, W, 3] RGB through jpeg_oracle's pixel path: what cv2.imdecode + BGR2RGB gives;
    `mistake` is passed to jpeg_oracle.idct_islow."""
    coef, hd = coefficients(blob)
    blk = coef.reshape(hd.mcuy, hd.mcux, hd.bpm, 64)
    c0, ups = 0, []
    for ci, (h, v) in enumerate(hd.samp):
        sel = blk[:, :, c0:c0 + h * v].reshape(-1, 64)
        px = JO.idct_islow(sel, hd.tables[ci][2], mistake).reshape(hd.mcuy, hd.mcux, v, h, 8, 8)
        pl = px.transpose(0, 2, 4, 1, 3, 5).reshape(hd.mcuy * v * 8, hd.mcux * h * 8)
        c0 += h * v
        dw, dh = -(-hd.width * h // hd.hmax), -(-hd.height * v // hd.vmax)
        ups.append(JO._upsample(pl, hd.hmax // h, hd.vmax // v, dw, dh, hd.height, hd.width))
    if hd.color == J.COLOR_GRAY:
        img = np.repeat(ups[0][..., None], 3, axis=2).astype(np.uint8)
    elif hd.color == J.COLOR_RGB:
        img = np.stack(ups, axis=-1).astype(np.uint8)
    else:
        img = JO._ycc_rgb(*ups)
    return np.ascontiguousarray(JO.orient(img, hd.orientation))
