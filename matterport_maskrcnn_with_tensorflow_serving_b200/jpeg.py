"""Host half of the device JPEG decoder (csrc/jpeg.cu, `mrx_jpeg_coefficients` / `mrx_jpeg_pixels`).

NumPy only.  `parse` walks a file's marker segments up to the start of its scan (the entropy-coded
bytes are never read here); `Plan` builds every image's Huffman lookups, quantisation tables,
geometry and device-buffer offsets, so that one upload describes the whole batch and every device
buffer is sized before anything runs.  `ProgressivePlan` does the same for progressive (SOF2) files
(`mrx_jpeg_progressive_coefficients`), and `plan_batch` routes each file of a batch by its frame
type.

What is accepted is what `cv2.imdecode(buf, IMREAD_COLOR)` (libjpeg-turbo, JDCT_ISLOW, fancy
upsampling) decodes bit for bit through the device path: baseline or extended sequential Huffman
(SOF0 / SOF1), 8-bit samples, 1 or 3 components in one interleaved scan, 8- or 16-bit quantisation
tables, restart intervals, integral sampling ratios with at most 10 blocks per MCU, EXIF orientation;
and progressive Huffman (SOF2) files with the same rules whose scan script is complete (every
coefficient sent and refined to Al = 0) and valid for libjpeg (no JERR_BAD_PROGRESSION, no
JWRN_BOGUS_PROGRESSION).  Anything else raises `JpegError` (a ValueError) naming the image's index and the reason.
"""
from __future__ import annotations

import numpy as np

from . import exif

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
    return exif.orientation(seg[6:])


class _Markers:
    """The marker-segment walk shared by `parse` and `ProgressivePlan`: the tables, restart interval,
    frame and colour hints in force at each SOS.  DHT, DQT and DRI may come again between the scans
    of a progressive file and replace what was defined before."""

    def __init__(self, data, fail):
        self.data, self.fail = data, fail
        self.qt, self.dc, self.ac = {}, {}, {}
        self.frame, self.ri, self.orientation = None, 0, 1
        self.jfif, self.adobe, self.exif_seen = False, None, False
        self.progressive = False

    def next_sos(self, pos):
        """Parse the segments from `pos` (a marker) up to the next SOS.  Returns (SOS payload, first
        byte after it), or (None, pos) when EOI comes first."""
        data, fail = self.data, self.fail
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
                return None, pos
            if pos + 2 > len(data):
                fail("truncated header")
            length = (data[pos] << 8) | data[pos + 1]
            if length < 2 or pos + length > len(data):
                fail("truncated header")
            seg = data[pos + 2:pos + length]
            pos += length
            if code in (0xC0, 0xC1, 0xC2):
                self._frame(seg)
                self.progressive = code == 0xC2
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
                    (self.dc if tc == 0 else self.ac)[th] = HuffTable(bits, vals, tc == 0, fail)
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
                    self.qt[tq] = tab
                    q += 1 + size
            elif code == 0xDD:
                if len(seg) < 2:
                    fail("truncated DRI")
                self.ri = (seg[0] << 8) | seg[1]
            elif code == 0xDC:
                fail("height defined by a DNL marker")
            elif code == 0xE0:
                if seg[:5] == b"JFIF\x00":
                    self.jfif = True
            elif code == 0xE1:
                o = _exif_orientation(seg)
                if o is not None and not self.exif_seen:      # the first Exif segment counts
                    self.orientation, self.exif_seen = o, True
            elif code == 0xEE:
                if len(seg) >= 12 and seg[:5] == b"Adobe":
                    self.adobe = seg[11]
            elif 0xE2 <= code <= 0xEF or code == 0xFE:
                pass
            elif code == 0xDA:
                return seg, pos
            else:
                fail(f"unsupported marker 0x{code:02X}")

    def _frame(self, seg):
        fail = self.fail
        if self.frame is not None:
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
        self.frame = (h, w, comps)

    def scan_components(self, seg):
        """The frame indices of an SOS payload's components, in frame order, and its (Ss, Se, Ah,
        Al) and (Td, Ta) selectors."""
        fail = self.fail
        comps = self.frame[2]
        if len(seg) < 1:
            fail("truncated scan header")
        ns = seg[0]
        if len(seg) < 1 + 2 * ns + 3:
            fail("truncated scan header")
        ids = [c[0] for c in comps]
        idx, sel = [], []
        for i in range(ns):
            cs, t = seg[1 + 2 * i], seg[2 + 2 * i]
            idx.append(ids.index(cs) if cs in ids else -1)
            sel.append((t >> 4, t & 15))
        ahal = seg[3 + 2 * ns]
        return idx, sel, (seg[1 + 2 * ns], seg[2 + 2 * ns], ahal >> 4, ahal & 15)

    def geometry(self):
        """Colour transform, sampling, MCU geometry and size checks of the frame."""
        fail = self.fail
        h, w, comps = self.frame
        if len(comps) == 1:
            color = COLOR_GRAY
            samp = [(1, 1)]
        else:
            if self.jfif:
                color = COLOR_YCC
            elif self.adobe is not None:
                color = COLOR_RGB if self.adobe == 0 else COLOR_YCC
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
        return dict(height=h, width=w, ncomp=len(comps), color=color,
                    orientation=self.orientation, samp=samp, hmax=hmax, vmax=vmax,
                    mcux=-(-w // (8 * hmax)), mcuy=-(-h // (8 * vmax)), bpm=bpm)

    def check_pixels(self):
        h, w, _ = self.frame
        if h * w > MAX_PIXELS:
            self.fail(f"{h}x{w} is more than {MAX_PIXELS} pixels (cv2.imdecode refuses it too)")


def _start(blob, index):
    data = bytes(blob)

    def fail(reason):
        raise JpegError(f"image {index}: {reason}")

    if len(data) < 4 or data[0] != 0xFF or data[1] != 0xD8:
        fail("not a JPEG file (no SOI marker)")
    if len(data) > MAX_FILE_BYTES:
        fail(f"file of {len(data)} bytes is larger than {MAX_FILE_BYTES}")
    mk = _Markers(data, fail)
    seg, pos = mk.next_sos(2)
    if seg is None:
        fail("no scan before EOI")
    if mk.frame is None:
        fail("no frame header before SOS")
    return data, fail, mk, seg, pos


def parse(blob, index=0):
    """Walk the marker segments of one JPEG file up to its first SOS.  Raises JpegError.

    A progressive (SOF2) file gives a Header with `progressive` set and its geometry only (no scan
    tables): `ProgressivePlan` walks the rest of it."""
    data, fail, mk, seg, pos = _start(blob, index)
    if mk.progressive:
        geo = mk.geometry()
        mk.check_pixels()
        return Header(**geo, restart_interval=mk.ri, scan_off=pos, file_len=len(data),
                      tables=None, progressive=True)
    comps = mk.frame[2]
    idx, sel, (ss, se, ah, al) = mk.scan_components(seg)
    if len(idx) != len(comps):
        fail("non-interleaved scan (more than one scan)")
    scomps = []
    for i, (ci, (td, ta)) in enumerate(zip(idx, sel)):
        if ci != i:
            fail("scan component order does not match the frame")
        if td not in mk.dc or ta not in mk.ac:
            fail("missing Huffman table")
        if comps[i][3] not in mk.qt:
            fail("missing quantisation table")
        scomps.append((mk.dc[td], mk.ac[ta], mk.qt[comps[i][3]]))
    if ss != 0 or se != 63 or ah != 0 or al != 0:
        fail("scan is not sequential (Ss, Se, Ah, Al)")
    geo = mk.geometry()
    if pos >= len(data):
        fail("truncated file (no scan data)")
    mk.check_pixels()
    blocks = geo["mcux"] * geo["mcuy"] * geo["bpm"]
    if 2 * blocks > 8 * (len(data) - pos):
        # every block takes at least two codes (DC, then AC or EOB) of at least one bit each
        fail(f"data ended before the last MCU ({len(data) - pos} bytes of scan for {blocks} "
             "blocks)")
    return Header(**geo, restart_interval=mk.ri, scan_off=pos, file_len=len(data),
                  tables=scomps, progressive=False)


def _as_bytes(blob, index):
    if isinstance(blob, (bytes, bytearray)):
        return bytes(blob)
    if isinstance(blob, memoryview):
        return blob.tobytes()
    raise TypeError(f"image {index}: expected bytes, bytearray or memoryview, got "
                    f"{type(blob).__name__}")


def _describe_pixels(D, hd, file_off, coef, planes):
    """The descriptor words `mrx_jpeg_pixels` reads (file, geometry, coefficient and plane
    offsets) for either plan.  Returns the next free plane offset."""
    D[D_FILE_OFF], D[D_FILE_LEN], D[D_SCAN_OFF] = file_off, hd.file_len, hd.scan_off
    D[D_H], D[D_W], D[D_NCOMP], D[D_COLOR] = hd.height, hd.width, hd.ncomp, hd.color
    D[D_ORIENT] = hd.orientation
    D[D_HMAX], D[D_VMAX], D[D_MCUX], D[D_MCUY] = hd.hmax, hd.vmax, hd.mcux, hd.mcuy
    D[D_BPM] = hd.bpm
    D[D_COEF_OFF], D[D_NBLOCKS] = coef, hd.mcux * hd.mcuy * hd.bpm
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
    return planes


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
        for i, hd in zip(index, self.headers):
            if hd.progressive:
                raise JpegError(f"image {i}: {_SOF_NAMES[0xC2]} frames are not supported by "
                                "jpeg.Plan (see ProgressivePlan)")
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
            D[D_RI], D[D_NUNITS] = ri, n_units
            D[D_UNST_OFF] = unst
            # work (int32): unit start bits [n_units+1], unit first subsequence [n_units+1],
            # then per subsequence: unit, exit bit, exit (block, zig-zag) state, blocks started,
            # then 3 words: the subsequence count, the sync rounds and the walk's re-decodes
            D[D_UNIT_BIT] = work
            D[D_UNIT_SUB] = work + n_units + 1
            D[D_SUB_OFF] = work + 2 * (n_units + 1)
            D[D_SUB_CAP] = sub_cap
            D[D_UNIT_BASE] = units
            planes = _describe_pixels(D, hd, file_off, coef, planes)
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


# ---- progressive files: int64 words per scan (csrc/jpeg.cu, the progressive section) ----
S_IMG, S_SS, S_SE, S_AH, S_AL, S_NCOMP, S_DATA_OFF, S_DATA_LEN, S_UNST_OFF = range(9)
S_UNIT_BIT, S_NUNITS, S_RI, S_NMCU, S_BW, S_TAB_OFF, S_UNIT_BASE, S_BPM = range(9, 17)
S_COMP, S_FIRST, S_H, S_V = 17, 20, 23, 26        # per component of the scan (3 words each)
SCAN_WORDS = 32
SCAN_TAB_BYTES = 3 * HUFF_BYTES     # per scan: the Huffman table of each component of the scan
MAX_SCANS = 256                   # mrx.h MRX_JPEG_MAX_SCANS: rounds of one decode
PROG_PAD = 32                     # zero bytes after each unstuffed scan (csrc/jpeg.cu kProgPad)


class Scan:
    """One scan of a progressive file: its frame components, spectral band and bit position, the
    byte range of its entropy-coded data, the restart interval in force and its Huffman tables."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _marker_starts(data):
    """The start of every run of 0xFF bytes followed by neither 0x00 nor RSTn (the 0xFF bytes
    before a marker are fill bytes): the first one at or after a scan's data is where the scan
    ends (the entropy-coded bytes are not read otherwise)."""
    a = np.frombuffer(data, dtype=np.uint8)
    ff = np.flatnonzero(a[:-1] == 0xFF)
    head = ff[(ff == 0) | (a[ff - 1] != 0xFF)]
    other = np.flatnonzero(a != 0xFF)
    j = np.searchsorted(other, head)
    nx = np.where(j < len(other), a[other[np.minimum(j, len(other) - 1)]], 0xD9)
    return head[(nx != 0x00) & ((nx < 0xD0) | (nx > 0xD7))]


def parse_progressive(blob, index=0):
    """Walk every marker segment of a progressive (SOF2) file.  Returns (Header, [Scan]) with the
    header's `tables` holding each component's quantisation table, latched at the first scan that
    contains the component (libjpeg's latch_quant_tables).  Raises JpegError for a bad
    (JERR_BAD_PROGRESSION) or bogus (JWRN_BOGUS_PROGRESSION) scan, or a script that leaves some
    coefficient unsent or unrefined (libjpeg-turbo would then smooth the blocks)."""
    data, fail, mk, seg, pos = _start(blob, index)
    if not mk.progressive:
        fail("not a progressive (SOF2) file")
    geo = mk.geometry()
    mk.check_pixels()
    comps = mk.frame[2]
    nc = len(comps)
    first = np.cumsum([0] + [h * v for h, v in geo["samp"]])
    marks = _marker_starts(data)
    coef_bits = np.full((nc, 64), -1, dtype=np.int32)
    quant = [None] * nc
    scans = []
    scan_off = pos
    while seg is not None:
        if len(scans) == MAX_SCANS:
            fail(f"more than {MAX_SCANS} scans")
        idx, sel, (ss, se, ah, al) = mk.scan_components(seg)
        if not idx or min(idx) < 0:
            fail("scan component not in the frame")
        if idx != sorted(set(idx)):
            fail("scan component order does not match the frame")
        bad = se != 0 if ss == 0 else (ss > se or se > 63 or len(idx) != 1)
        if (ah and al != ah - 1) or al > 13 or bad:
            fail(f"bad progression (Ss={ss}, Se={se}, Ah={ah}, Al={al})")
        for ci in idx:
            if ss and coef_bits[ci, 0] < 0:
                fail(f"bogus progression (an AC scan of component {ci} before its DC scan)")
            for k in range(ss, se + 1):
                want = max(int(coef_bits[ci, k]), 0)
                if ah != want:
                    fail(f"bogus progression (component {ci}, coefficient {k}: Ah={ah}, "
                         f"expected {want})")
            coef_bits[ci, ss:se + 1] = al
            if quant[ci] is None:
                if comps[ci][3] not in mk.qt:
                    fail("missing quantisation table")
                quant[ci] = mk.qt[comps[ci][3]].copy()
        tables = []
        for td, ta in sel:
            if ss == 0 and ah == 0 and td not in mk.dc or ss and ta not in mk.ac:
                fail("missing Huffman table")
            tables.append(mk.dc[td] if ss == 0 and ah == 0 else mk.ac[ta] if ss else None)
        k = int(np.searchsorted(marks, pos))
        if k == len(marks):
            fail("truncated file (no marker after a scan)")
        end = int(marks[k])
        if len(idx) > 1:
            nmcu, bw = geo["mcux"] * geo["mcuy"], geo["mcux"]
        else:
            h, v = geo["samp"][idx[0]]
            bw = -(-(-(-geo["width"] * h // geo["hmax"])) // 8)
            nmcu = bw * -(-(-(-geo["height"] * v // geo["vmax"])) // 8)
        ri = mk.ri or nmcu
        scans.append(Scan(comps=idx, ss=ss, se=se, ah=ah, al=al, tables=tables, data_off=pos,
                          data_len=end - pos, ri=ri, nmcu=nmcu, bw=bw, units=-(-nmcu // ri),
                          first=[int(first[ci]) for ci in idx],
                          samp=[geo["samp"][ci] if len(idx) > 1 else (1, 1) for ci in idx]))
        seg, pos = mk.next_sos(end)
    if (coef_bits != 0).any():
        ci, k = np.argwhere(coef_bits != 0)[0]
        fail(f"incomplete progressive script (component {ci}, coefficient {k} ends at "
             f"Al={coef_bits[ci, k]}; only complete scripts are supported)")
    hd = Header(**geo, restart_interval=scans[0].ri, scan_off=scan_off, file_len=len(data),
                tables=[(None, None, q) for q in quant], progressive=True)
    return hd, scans


def _pack_quant(hd):
    out = np.zeros(TAB_BYTES, dtype=np.uint8)
    for ci, (_, _, q) in enumerate(hd.tables):
        o = ci * COMP_TAB_BYTES
        out[o:o + 256] = np.frombuffer(q.astype(np.int32).tobytes(), dtype=np.uint8)
    return out


def scan_levels(scans):
    """The round of each scan of one file: one more than the latest round of an earlier scan that
    shares a component and a coefficient with it (a refinement reads what that scan wrote), else 0.
    Scans of one round write disjoint coefficients, so they decode concurrently: in cv2's script
    every first scan is round 0, the first refinements round 1 and the last luma refinement round 2."""
    lv = []
    for i, sc in enumerate(scans):
        lv.append(max([lv[j] + 1 for j, o in enumerate(scans[:i])
                       if set(o.comps) & set(sc.comps) and o.ss <= sc.se and sc.ss <= o.se],
                      default=0))
    return lv


class ProgressivePlan:
    """A batch of progressive files laid out for the device (`mrx_jpeg_progressive_coefficients`,
    then `mrx_jpeg_pixels` as for `Plan`): the files, the 80-word image descriptors and quantisation
    tables `mrx_jpeg_pixels` reads, one SCAN_WORDS descriptor and Huffman table blob per scan, and
    the restart units of every scan grouped by round.  A scan's round is its dependency level
    (`scan_levels`): it runs after the earlier scans of its image that touch the same coefficients,
    and with every scan that does not.  Sizes depend on the headers and the byte lengths of the
    scans only."""

    def __init__(self, blobs, index=None):
        index = list(range(len(blobs))) if index is None else list(index)
        datas = [_as_bytes(b, i) for i, b in zip(index, blobs)]
        parsed = [parse_progressive(d, i) for i, d in zip(index, datas)]
        self.headers = [hd for hd, _ in parsed]
        self.scans = [sc for _, sc in parsed]
        B = self.B = len(datas)
        desc = np.zeros((B, DESC_WORDS), dtype=np.int64)
        tabs = np.zeros((B, TAB_BYTES), dtype=np.uint8)
        file_off = coef = planes = 0
        self.max_blocks = self.max_pixels = 1
        for b, hd in enumerate(self.headers):
            planes = _describe_pixels(desc[b], hd, file_off, coef, planes)
            tabs[b] = _pack_quant(hd)
            file_off += _align(hd.file_len, 16)
            coef += int(desc[b, D_NBLOCKS])
            self.max_blocks = max(self.max_blocks, int(desc[b, D_NBLOCKS]))
            self.max_pixels = max(self.max_pixels, hd.height * hd.width)
        levels = [scan_levels(s) for s in self.scans]
        R = self.rounds = max((max(lv) + 1 for lv in levels), default=0)
        order = [(r, b, i) for r in range(R) for b in range(B)
                 for i in range(len(levels[b])) if levels[b][i] == r]
        n = self.n_scans = len(order)
        sd = np.zeros((max(n, 1), SCAN_WORDS), dtype=np.int64)
        stabs = np.zeros((max(n, 1), SCAN_TAB_BYTES), dtype=np.uint8)
        unit_scan, round_off = [], [0] * (R + 1)
        unst = unit_bit = 0
        for j, (r, b, i) in enumerate(order):
            sc, W = self.scans[b][i], sd[j]
            W[S_IMG], W[S_SS], W[S_SE], W[S_AH], W[S_AL] = b, sc.ss, sc.se, sc.ah, sc.al
            W[S_NCOMP] = len(sc.comps)
            W[S_DATA_OFF], W[S_DATA_LEN] = desc[b, D_FILE_OFF] + sc.data_off, sc.data_len
            W[S_UNST_OFF], W[S_UNIT_BIT], W[S_NUNITS] = unst, unit_bit, sc.units
            W[S_RI], W[S_NMCU], W[S_BW], W[S_TAB_OFF] = sc.ri, sc.nmcu, sc.bw, j * SCAN_TAB_BYTES
            W[S_UNIT_BASE] = len(unit_scan)
            W[S_BPM] = sum(h * v for h, v in sc.samp)
            for i, ci in enumerate(sc.comps):
                h, v = self.headers[b].samp[ci]
                W[S_COMP + i], W[S_FIRST + i] = ci, sc.first[i]
                W[S_H + i], W[S_V + i] = h, v
                if sc.tables[i] is not None:
                    o = i * HUFF_BYTES
                    stabs[j, o:o + HUFF_BYTES] = np.frombuffer(sc.tables[i].pack(), np.uint8)
            unit_scan.extend([j] * sc.units)
            round_off[r + 1] = len(unit_scan)
            unst += _align(sc.data_len + PROG_PAD, 16)
            unit_bit += sc.units + 1
        files = np.zeros(max(file_off, 16), dtype=np.uint8)
        for b, d in enumerate(datas):
            o = int(desc[b, D_FILE_OFF])
            files[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
        self.files, self.desc, self.tabs = files, desc, tabs
        self.scan_desc, self.scan_tabs = sd, stabs
        self.unit_scan = np.asarray(unit_scan or [0], dtype=np.int32)
        self.round_off = np.asarray(round_off, dtype=np.int32)
        self.max_round_units = max([int(round_off[r + 1] - round_off[r]) for r in range(R)] + [1])
        self.unst_bytes = max(unst, 16)
        self.unit_bit_words = max(unit_bit, 1)
        self.coef_blocks = max(coef, 1)
        self.plane_bytes = max(planes, 16)
        self.shapes = [hd.shape for hd in self.headers]


def _frame_marker(data):
    """The SOFn code of a file found by skipping segments by their lengths (no payload is read),
    or None.  Only routes the file: the plan it goes to parses it and refuses what is wrong."""
    pos = 2
    while pos + 4 <= len(data) and data[pos] == 0xFF:
        code = data[pos + 1]
        if 0xC0 <= code <= 0xCF and code not in (0xC4, 0xC8, 0xCC):
            return code
        if code == 0xFF:
            pos += 1
            continue
        if code in (0xD8, 0x01) or 0xD0 <= code <= 0xD7:
            pos += 2
            continue
        if code in (0xD9, 0xDA):
            return None
        pos += 2 + ((data[pos + 2] << 8) | data[pos + 3])
    return None


def plan_batch(blobs, index=None, S=DEFAULT_S):
    """A batch of files split by frame type: ([(Plan or ProgressivePlan, positions in blobs)],
    the decoded shape of every file).  Sequential files go to one `Plan`, progressive ones to one
    `ProgressivePlan`; each keeps the caller's index for its refusals."""
    index = list(range(len(blobs))) if index is None else list(index)
    datas = [_as_bytes(b, i) for i, b in zip(index, blobs)]
    prog = [_frame_marker(d) == 0xC2 for d in datas]
    plans, shapes = [], [None] * len(datas)
    for want, make in ((False, lambda ds, ix: Plan(ds, S, index=ix)),
                       (True, lambda ds, ix: ProgressivePlan(ds, index=ix))):
        pos = [k for k, p in enumerate(prog) if p == want]
        if pos:
            plan = make([datas[k] for k in pos], [index[k] for k in pos])
            plans.append((plan, pos))
            for k, sh in zip(pos, plan.shapes):
                shapes[k] = sh
    return plans, shapes


def status_reasons(bits):
    """Reasons for a nonzero device status word (mrx.h MRX_JPEG_ST_*)."""
    names = [(1, "bad Huffman code"), (2, "data ended before the last MCU"),
             (4, "missing or out-of-order RST marker"), (8, "DC coefficient overflows int32"),
             (16, "a marker other than EOI or RSTn inside or after the scan")]
    return ", ".join(n for bit, n in names if bits & bit)
