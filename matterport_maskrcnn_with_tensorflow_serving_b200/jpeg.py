"""Host half of the device JPEG decoder (csrc/jpeg.cu, `mrx_jpeg_coefficients` / `mrx_jpeg_pixels`).

NumPy only.  `parse` walks a file's marker segments up to the start of its scan (the entropy-coded
bytes are never read here); `Plan` builds every image's Huffman lookups, quantisation tables,
geometry and device-buffer offsets, so that one upload describes the whole batch and every device
buffer is sized before anything runs.

What is accepted is what `cv2.imdecode(buf, IMREAD_COLOR)` (libjpeg-turbo, JDCT_ISLOW, fancy
upsampling) decodes bit for bit through the device path: baseline or extended sequential Huffman
(SOF0 / SOF1), 8-bit samples, 1 or 3 components in one interleaved scan, 8- or 16-bit quantisation
tables, restart intervals, integral sampling ratios with at most 10 blocks per MCU, EXIF orientation.
Anything else raises `JpegError` (a ValueError) naming the image's index and the reason.
"""
from __future__ import annotations

import struct

import numpy as np

# zig-zag index -> natural (row-major) index, with libjpeg's 16 guard entries for a corrupt run
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27,
    20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58,
    59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63] + [63] * 16, dtype=np.int32)

MAX_BLOCKS_PER_MCU = 10
MAX_FILE_BYTES = 1 << 27          # keeps every bit position of an image in int32
MAX_PIXELS = 1 << 30              # cv2's CV_IO_MAX_IMAGE_PIXELS: imdecode refuses larger images
FAST_BITS = 9
DEFAULT_S = 1024                   # bits per subsequence of the self-synchronising decode

COLOR_GRAY, COLOR_YCC, COLOR_RGB = 0, 1, 2

# ---- the device descriptor: int64 words per image (csrc/jpeg.cu, struct field indices) ----
D_FILE_OFF, D_FILE_LEN, D_SCAN_OFF, D_H, D_W, D_NCOMP, D_COLOR, D_ORIENT = range(8)
D_HMAX, D_VMAX, D_MCUX, D_MCUY, D_BPM, D_RI, D_NUNITS = range(8, 15)
D_UNST_OFF, D_UNIT_BIT, D_UNIT_SUB, D_SUB_OFF, D_SUB_CAP, D_COEF_OFF, D_NBLOCKS = range(15, 22)
D_PLANE_OFF, D_COMP_H, D_COMP_V, D_PLANE_BW, D_PLANE_BH, D_DW, D_DH = 22, 25, 28, 31, 34, 37, 40
D_BLK_COMP, D_BLK_DX, D_BLK_DY = 43, 53, 63
D_UNIT_BASE = 73                    # the image's first entry in the batch's unit -> image table
DESC_WORDS = 80
WORK_TAIL = 3                       # per image after its subsequences (see Plan)

# ---- the table blob: per image, per component: quant int32[64] (natural order), DC and AC tables
HUFF_BYTES = 2 * (1 << FAST_BITS) + 4 * 18 + 4 * 18 + 256      # lookup u16, maxcode, valptr, vals
COMP_TAB_BYTES = 4 * 64 + 2 * HUFF_BYTES
TAB_BYTES = 3 * COMP_TAB_BYTES

_SOF_NAMES = {0xC2: "progressive (SOF2)", 0xC3: "lossless (SOF3)", 0xC5: "hierarchical (SOF5)",
              0xC6: "hierarchical (SOF6)", 0xC7: "hierarchical (SOF7)",
              0xC9: "arithmetic-coded (SOF9)", 0xCA: "arithmetic-coded (SOF10)",
              0xCB: "arithmetic-coded (SOF11)", 0xCD: "arithmetic-coded (SOF13)",
              0xCE: "arithmetic-coded (SOF14)", 0xCF: "arithmetic-coded (SOF15)"}


class JpegError(ValueError):
    """A file the device decoder does not accept (or whose entropy-coded data is corrupt)."""


class HuffTable:
    """One DHT table: libjpeg's canonical codes, a FAST_BITS lookup and maxcode / valptr."""

    def __init__(self, bits, vals, is_dc, fail):
        bits = [int(b) for b in bits]
        vals = [int(v) for v in vals]
        self.bits, self.vals = bits, vals
        if is_dc and any(v > 15 for v in vals):
            fail("bogus Huffman table (DC symbol above 15)")
        lookup = np.zeros(1 << FAST_BITS, dtype=np.uint16)
        maxcode = np.full(18, -1, dtype=np.int32)
        valptr = np.zeros(18, dtype=np.int32)
        code, k = 0, 0
        for length in range(1, 17):
            n = bits[length - 1]
            if n:
                valptr[length] = k - code
                for _ in range(n):
                    if length <= FAST_BITS:
                        lo = code << (FAST_BITS - length)
                        lookup[lo:lo + (1 << (FAST_BITS - length))] = (length << 8) | vals[k]
                    code += 1
                    k += 1
                maxcode[length] = code - 1
            if code >= (1 << length):
                fail("bogus Huffman table (code space overflow)")
            code <<= 1
        maxcode[17] = 0x7FFFFFFF
        self.lookup, self.maxcode, self.valptr = lookup, maxcode, valptr

    def pack(self):
        vals = np.zeros(256, dtype=np.uint8)
        vals[:len(self.vals)] = self.vals
        return (self.lookup.tobytes() + self.maxcode.tobytes() + self.valptr.tobytes() +
                vals.tobytes())


class Header:
    """What `parse` found: frame, tables in use, scan start, orientation and geometry."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    @property
    def shape(self):
        """(H, W, 3) of the decoded, oriented image."""
        if self.orientation >= 5:
            return (self.width, self.height, 3)
        return (self.height, self.width, 3)


def _exif_orientation(seg):
    """IFD0 tag 0x0112 of an APP1 Exif payload, or 1."""
    if len(seg) < 14 or seg[:6] != b"Exif\x00\x00":
        return None
    t = seg[6:]
    if t[:2] == b"II":
        e = "<"
    elif t[:2] == b"MM":
        e = ">"
    else:
        return 1
    try:
        if struct.unpack(e + "H", t[2:4])[0] != 42:
            return 1
        ifd = struct.unpack(e + "I", t[4:8])[0]
        n = struct.unpack(e + "H", t[ifd:ifd + 2])[0]
        for i in range(n):
            p = ifd + 2 + 12 * i
            tag, typ, cnt = struct.unpack(e + "HHI", t[p:p + 8])
            if tag == 0x0112 and typ == 3:
                v = struct.unpack(e + "H", t[p + 8:p + 10])[0]
                return v if 1 <= v <= 8 else 1
    except struct.error:
        return 1
    return 1


def parse(blob, index=0):
    """Walk the marker segments of one JPEG file up to its SOS.  Raises JpegError."""
    data = bytes(blob)

    def fail(reason):
        raise JpegError(f"image {index}: {reason}")

    if len(data) < 4 or data[0] != 0xFF or data[1] != 0xD8:
        fail("not a JPEG file (no SOI marker)")
    if len(data) > MAX_FILE_BYTES:
        fail(f"file of {len(data)} bytes is larger than {MAX_FILE_BYTES}")
    qt, dc, ac = {}, {}, {}
    frame, ri, orientation = None, 0, 1
    jfif, adobe, exif_seen = False, None, False
    pos = 2
    while True:
        if pos + 2 > len(data):
            fail("truncated header (no SOS marker)")
        if data[pos] != 0xFF:
            fail(f"bogus marker at byte {pos}")
        while pos < len(data) and data[pos] == 0xFF:
            pos += 1
        if pos >= len(data):
            fail("truncated header")
        code = data[pos]
        pos += 1
        if code in (0x01,) or 0xD0 <= code <= 0xD7:
            continue
        if code == 0xD9:
            fail("no scan before EOI")
        if pos + 2 > len(data):
            fail("truncated header")
        length = (data[pos] << 8) | data[pos + 1]
        if length < 2 or pos + length > len(data):
            fail("truncated header")
        seg = data[pos + 2:pos + length]
        pos += length
        if code in (0xC0, 0xC1):
            if frame is not None:
                fail("two frame headers")
            if len(seg) < 6:
                fail("truncated frame header")
            p, h, w, n = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if p != 8:
                fail(f"{p}-bit samples (only 8-bit is supported)")
            if h == 0:
                fail("height defined by a DNL marker")
            if w == 0:
                fail("image width 0")
            if n not in (1, 3):
                fail(f"{n} components (only 1 or 3 are supported)")
            if len(seg) < 6 + 3 * n:
                fail("truncated frame header")
            comps = []
            for i in range(n):
                cid, hv, tq = seg[6 + 3 * i], seg[7 + 3 * i], seg[8 + 3 * i]
                hs, vs = hv >> 4, hv & 15
                if not (1 <= hs <= 4 and 1 <= vs <= 4) or tq > 3:
                    fail("bogus sampling factors or quantisation table index")
                comps.append((cid, hs, vs, tq))
            frame = (h, w, comps)
        elif code in _SOF_NAMES:
            fail(f"{_SOF_NAMES[code]} frames are not supported")
        elif code == 0xCC:
            fail("arithmetic-coded (DAC) frames are not supported")
        elif code == 0xC4:
            q = 0
            while q < len(seg):
                if q + 17 > len(seg):
                    fail("bogus Huffman table (truncated DHT)")
                tc, th = seg[q] >> 4, seg[q] & 15
                bits = list(seg[q + 1:q + 17])
                count = sum(bits)
                if tc > 1 or th > 3 or count > 256 or q + 17 + count > len(seg):
                    fail("bogus Huffman table")
                vals = list(seg[q + 17:q + 17 + count])
                (dc if tc == 0 else ac)[th] = HuffTable(bits, vals, tc == 0, fail)
                q += 17 + count
        elif code == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                size = 64 * (2 if pq else 1)
                if pq > 1 or tq > 3 or q + 1 + size > len(seg):
                    fail("bogus quantisation table")
                raw = np.frombuffer(seg[q + 1:q + 1 + size], dtype=">u2" if pq else np.uint8)
                tab = np.zeros(64, dtype=np.int32)
                tab[ZIGZAG[:64]] = raw
                qt[tq] = tab
                q += 1 + size
        elif code == 0xDD:
            if len(seg) < 2:
                fail("truncated DRI")
            ri = (seg[0] << 8) | seg[1]
        elif code == 0xDC:
            fail("height defined by a DNL marker")
        elif code == 0xE0:
            if seg[:5] == b"JFIF\x00":
                jfif = True
        elif code == 0xE1:
            o = _exif_orientation(seg)
            if o is not None and not exif_seen:      # the first Exif segment counts
                orientation, exif_seen = o, True
        elif code == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe = seg[11]
        elif 0xE2 <= code <= 0xEF or code == 0xFE:
            pass
        elif code == 0xDA:
            break
        else:
            fail(f"unsupported marker 0x{code:02X}")
    if frame is None:
        fail("no frame header before SOS")
    h, w, comps = frame
    if len(seg) < 1:
        fail("truncated scan header")
    ns = seg[0]
    if len(seg) < 1 + 2 * ns + 3:
        fail("truncated scan header")
    if ns != len(comps):
        fail("non-interleaved scan (more than one scan)")
    scomps = []
    for i in range(ns):
        cs, t = seg[1 + 2 * i], seg[2 + 2 * i]
        ci = [c[0] for c in comps].index(cs) if cs in [c[0] for c in comps] else -1
        if ci != i:
            fail("scan component order does not match the frame")
        td, ta = t >> 4, t & 15
        if td not in dc or ta not in ac:
            fail("missing Huffman table")
        if comps[i][3] not in qt:
            fail("missing quantisation table")
        scomps.append((dc[td], ac[ta], qt[comps[i][3]]))
    ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
    if ss != 0 or se != 63 or ahal != 0:
        fail("scan is not sequential (Ss, Se, Ah, Al)")
    if len(comps) == 1:
        color = COLOR_GRAY
        samp = [(1, 1)]
    else:
        if jfif:
            color = COLOR_YCC
        elif adobe is not None:
            color = COLOR_RGB if adobe == 0 else COLOR_YCC
        elif [c[0] for c in comps] == [82, 71, 66]:
            color = COLOR_RGB
        else:
            color = COLOR_YCC
        samp = [(c[1], c[2]) for c in comps]
    hmax = max(s[0] for s in samp)
    vmax = max(s[1] for s in samp)
    if any(hmax % s[0] or vmax % s[1] for s in samp):
        fail("non-integral sampling ratios")
    bpm = sum(s[0] * s[1] for s in samp)
    if bpm > MAX_BLOCKS_PER_MCU:
        fail(f"{bpm} blocks per MCU (at most {MAX_BLOCKS_PER_MCU})")
    if pos >= len(data):
        fail("truncated file (no scan data)")
    if h * w > MAX_PIXELS:
        fail(f"{h}x{w} is more than {MAX_PIXELS} pixels (cv2.imdecode refuses it too)")
    mcux = -(-w // (8 * hmax))
    mcuy = -(-h // (8 * vmax))
    blocks = mcux * mcuy * bpm
    if 2 * blocks > 8 * (len(data) - pos):
        # every block takes at least two codes (DC, then AC or EOB) of at least one bit each
        fail(f"data ended before the last MCU ({len(data) - pos} bytes of scan for {blocks} "
             "blocks)")
    return Header(height=h, width=w, ncomp=len(comps), color=color, orientation=orientation,
                  samp=samp, hmax=hmax, vmax=vmax, mcux=mcux, mcuy=mcuy, bpm=bpm,
                  restart_interval=ri, scan_off=pos, file_len=len(data), tables=scomps)


def _as_bytes(blob, index):
    if isinstance(blob, (bytes, bytearray)):
        return bytes(blob)
    if isinstance(blob, memoryview):
        return blob.tobytes()
    raise TypeError(f"image {index}: expected bytes, bytearray or memoryview, got "
                    f"{type(blob).__name__}")


def _pack_tables(hd):
    out = bytearray()
    for ci in range(3):
        if ci < len(hd.tables):
            d, a, q = hd.tables[ci]
            out += q.astype(np.int32).tobytes() + d.pack() + a.pack()
        else:
            out += bytes(COMP_TAB_BYTES)
    assert len(out) == TAB_BYTES
    return bytes(out)


def _align(n, a):
    return -(-n // a) * a


class Plan:
    """One batch of files laid out for the device: the upload (files, desc, tabs, unit_img) and
    the sizes of every device buffer.  Sizes depend on the headers and the file lengths only."""

    def __init__(self, blobs, S=DEFAULT_S, index=None):
        if S < 32 or S % 32 or S > (1 << 16):
            raise ValueError(f"S={S}: a multiple of 32 in [32, 65536]")
        self.S = int(S)
        index = list(range(len(blobs))) if index is None else list(index)
        datas = [_as_bytes(b, i) for i, b in zip(index, blobs)]
        self.headers = [parse(d, i) for i, d in zip(index, datas)]
        B = len(datas)
        self.B = B
        desc = np.zeros((B, DESC_WORDS), dtype=np.int64)
        tabs = np.zeros((B, TAB_BYTES), dtype=np.uint8)
        file_off = unst = work = coef = planes = units = 0
        unit_img = []
        self.max_subs = self.max_blocks = self.max_pixels = 1
        for b, (d, hd) in enumerate(zip(datas, self.headers)):
            D = desc[b]
            scan_len = hd.file_len - hd.scan_off
            mcus = hd.mcux * hd.mcuy
            ri = hd.restart_interval if hd.restart_interval else mcus
            n_units = -(-mcus // ri)
            sub_cap = -(-scan_len * 8 // self.S) + n_units
            n_blocks = mcus * hd.bpm
            D[D_FILE_OFF], D[D_FILE_LEN], D[D_SCAN_OFF] = file_off, hd.file_len, hd.scan_off
            D[D_H], D[D_W], D[D_NCOMP], D[D_COLOR] = hd.height, hd.width, hd.ncomp, hd.color
            D[D_ORIENT] = hd.orientation
            D[D_HMAX], D[D_VMAX], D[D_MCUX], D[D_MCUY] = hd.hmax, hd.vmax, hd.mcux, hd.mcuy
            D[D_BPM], D[D_RI], D[D_NUNITS] = hd.bpm, ri, n_units
            D[D_UNST_OFF] = unst
            # work (int32): unit start bits [n_units+1], unit first subsequence [n_units+1],
            # then per subsequence: unit, exit bit, exit (block, zig-zag) state, blocks started,
            # then 3 words: the subsequence count, the sync rounds and the walk's re-decodes
            D[D_UNIT_BIT] = work
            D[D_UNIT_SUB] = work + n_units + 1
            D[D_SUB_OFF] = work + 2 * (n_units + 1)
            D[D_SUB_CAP] = sub_cap
            D[D_COEF_OFF], D[D_NBLOCKS] = coef, n_blocks
            D[D_UNIT_BASE] = units
            c = 0
            for ci, (hs, vs) in enumerate(hd.samp):
                bw, bh = hd.mcux * hs, hd.mcuy * vs
                D[D_PLANE_OFF + ci] = planes
                D[D_COMP_H + ci], D[D_COMP_V + ci] = hs, vs
                D[D_PLANE_BW + ci], D[D_PLANE_BH + ci] = bw, bh
                D[D_DW + ci] = -(-hd.width * hs // hd.hmax)
                D[D_DH + ci] = -(-hd.height * vs // hd.vmax)
                planes += _align(bw * bh * 64, 16)
                for dy in range(vs):
                    for dx in range(hs):
                        D[D_BLK_COMP + c], D[D_BLK_DX + c], D[D_BLK_DY + c] = ci, dx, dy
                        c += 1
            tabs[b] = np.frombuffer(_pack_tables(hd), dtype=np.uint8)
            unit_img.extend([b] * n_units)
            file_off += _align(hd.file_len, 16)
            unst += _align(scan_len + 8, 16)
            work += 2 * (n_units + 1) + 4 * sub_cap + WORK_TAIL
            coef += n_blocks
            units += n_units
            self.max_subs = max(self.max_subs, sub_cap)
            self.max_blocks = max(self.max_blocks, n_blocks)
            self.max_pixels = max(self.max_pixels, hd.height * hd.width)
        files = np.zeros(max(file_off, 16), dtype=np.uint8)
        for b, d in enumerate(datas):
            o = int(desc[b, D_FILE_OFF])
            files[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
        self.files, self.desc, self.tabs = files, desc, tabs
        self.unit_img = np.asarray(unit_img if unit_img else [0], dtype=np.int32)
        self.units = units
        self.unst_bytes = max(unst, 16)
        self.work_words = max(work, 1)
        self.coef_blocks = max(coef, 1)
        self.plane_bytes = max(planes, 16)
        self.shapes = [hd.shape for hd in self.headers]


def status_reasons(bits):
    """Reasons for a nonzero device status word (mrx.h MRX_JPEG_ST_*)."""
    names = [(1, "bad Huffman code"), (2, "data ended before the last MCU"),
             (4, "missing or out-of-order RST marker"), (8, "DC coefficient overflows int32"),
             (16, "a marker other than EOI or RSTn inside or after the scan")]
    return ", ".join(n for bit, n in names if bits & bit)
