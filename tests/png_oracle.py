"""CPU restatement of the device PNG encoder (csrc/png.cu): what `cv2.imwrite(path, rgb[..., ::-1])`
writes for a uint8 RGB image, computed the way the kernels compute it.

libpng (as OpenCV calls it) filters every row with Sub (bpp 3; width-1 rows are stored unfiltered
with filter byte 0) and hands the rows one by one to zlib at level 1, strategy Z_RLE, memLevel 8.
zlib's run parse and block coding are restated here step for step:

- `parse`: position i of the filtered stream starts a symbol or not.  A stretch is a maximal run of
  bytes equal to their predecessor; a stretch of L bytes is floor(L/258) matches of 258 at distance
  1, then one match of the remainder r when r >= 3, else r literals.  Every other byte is a
  literal.  The per-position code is the device's `sym` array: -1 (inside a match), the literal
  byte 0..255, or 256 + length - 3 for a match.
- `blocks`: a block ends after 16383 symbols; the final block (last = 1) is flushed even when
  empty.  A block may be stored only while its bytes are still in zlib's sliding window
  (`stored_ok`), which depends on where the window slid (`slide_count`).
- `block_trees`: trees.c's build_tree (heap order, depth tiebreak), gen_bitlen (length-limit
  fix), gen_codes, scan_tree / send_tree and the stored / static / dynamic choice.
- the bit writer, Adler-32 (per-tile partial sums combined mod 65521), the zlib header with
  cv2's window bits, 8192-byte IDAT chunks with CRC-32, IHDR and IEND.
"""
from __future__ import annotations

import struct
import zlib

import numpy as np

MAX_MATCH = 258
SYMS_PER_BLOCK = 16383           # lit_bufsize - 1 at memLevel 8
IDAT_BYTES = 8192
L_CODES, D_CODES, BL_CODES = 286, 30, 19
HEAP_SIZE = 2 * L_CODES + 1
END_BLOCK = 256
STORED, STATIC, DYNAMIC = 0, 1, 2
TILE = 2048                      # positions per tile of the device scans

EXTRA_LBITS = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
EXTRA_DBITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11,
               12, 12, 13, 13]
EXTRA_BLBITS = [0] * 16 + [2, 3, 7]
BL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
BASE_LENGTH = [0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 32, 40, 48, 56, 64, 80, 96,
               112, 128, 160, 192, 224, 255]


def length_code(lc):
    """Length code index 0..28 of lc = match length - 3 (zlib's _length_code)."""
    if lc == 255:
        return 28
    for code in range(27, -1, -1):
        if lc >= BASE_LENGTH[code]:
            return code
    raise AssertionError


LENGTH_CODE = np.array([length_code(lc) for lc in range(256)], dtype=np.int32)
LENGTH_XBITS = np.array([EXTRA_LBITS[c] for c in LENGTH_CODE], dtype=np.int32)
LENGTH_XVAL = np.array([lc - BASE_LENGTH[c] for lc, c in enumerate(LENGTH_CODE)], dtype=np.int64)


def bi_reverse(code, n):
    r = 0
    for _ in range(n):
        r = (r << 1) | (code & 1)
        code >>= 1
    return r


def gen_codes(lens, max_code):
    """Canonical, bit-reversed codes for code lengths lens[0..max_code] (zlib's gen_codes)."""
    bl_count = [0] * 16
    for n in range(max_code + 1):
        bl_count[lens[n]] += 1
    bl_count[0] = 0
    next_code, code = [0] * 16, 0
    for bits in range(1, 16):
        code = (code + bl_count[bits - 1]) << 1
        next_code[bits] = code
    codes = [0] * len(lens)
    for n in range(max_code + 1):
        ln = lens[n]
        if ln:
            codes[n] = bi_reverse(next_code[ln], ln)
            next_code[ln] += 1
    return codes


STATIC_LLEN = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
STATIC_LCODE = gen_codes(STATIC_LLEN, 287)
STATIC_DLEN = [5] * 30
STATIC_DCODE = [bi_reverse(n, 5) for n in range(30)]


# ----------------------------------------------------------------------------- rows and header
def filter_rows(img):
    """uint8 [H, W, 3] RGB -> the filtered stream, H rows of (filter byte, 3W bytes)."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    H, W, _ = img.shape
    rows = img.reshape(H, 3 * W)
    out = np.empty((H, 3 * W + 1), dtype=np.uint8)
    if W == 1:
        out[:, 0] = 0
        out[:, 1:] = rows
    else:
        out[:, 0] = 1
        out[:, 1:4] = rows[:, :3]
        out[:, 4:] = rows[:, 3:] - rows[:, :-3]     # wraps mod 256
    return out.reshape(-1)


def window_bits(n):
    """(bits in the zlib header, windowBits zlib runs with) for an n-byte filtered stream."""
    wb, half = 15, 16384
    while n <= half and wb > 8:
        half >>= 1
        wb -= 1
    return wb, max(wb, 9)


def zlib_header(n):
    wb, _ = window_bits(n)
    cmf = ((wb - 8) << 4) | 8
    flg = 31 - (cmf << 8) % 31
    return bytes([cmf, flg])


def adler32(stream, tile=TILE):
    """Adler-32 as the device forms it: per tile, sum(s) and sum((n - i) * s) mod 65521, added."""
    n = len(stream)
    s = stream.astype(np.int64)
    w = (n - np.arange(n, dtype=np.int64)) % 65521
    acc_a = acc_b = 0
    for t in range(0, n, tile):
        acc_a += int(s[t:t + tile].sum()) % 65521
        acc_b += int((s[t:t + tile] * w[t:t + tile] % 65521).sum()) % 65521
    a = (1 + acc_a) % 65521
    b = (n + acc_b) % 65521
    return (b << 16) | a


def deflate_bound(n):
    """Worst-case deflate bytes for an n-byte stream: every block either static (<= 9 bits a byte
    plus 10 bits) or stored (8 bits a byte plus at most 42), at most n // 16383 + 2 blocks."""
    return (9 * n + 42 * (n // SYMS_PER_BLOCK + 2) + 7) // 8


def png_bound(n):
    z = 2 + deflate_bound(n) + 4
    return 8 + 25 + z + 12 * (-(-z // IDAT_BYTES)) + 12


def chunk(tag, data):
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data))


def ihdr(h, w):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))


# ----------------------------------------------------------------------------- parse
def parse(stream):
    """Per-position symbol code (the device's sym array): -1, 0..255 literal, 256 + len - 3."""
    s = np.asarray(stream, dtype=np.uint8)
    n = len(s)
    sym = s.astype(np.int16)
    eq = np.zeros(n, dtype=bool)
    eq[1:] = s[1:] == s[:-1]
    d = np.diff(np.concatenate([[0], eq.view(np.int8), [0]]))
    starts, ends = np.flatnonzero(d == 1), np.flatnonzero(d == -1)
    if len(starts) == 0:
        return sym
    lens = ends - starts
    sid = np.cumsum((d == 1)[:n]) - 1
    idx = np.flatnonzero(eq)
    st = starts[sid[idx]]
    L = lens[sid[idx]]
    j = idx - st
    full = (L // MAX_MATCH) * MAX_MATCH
    r = L - full
    code = s[idx].astype(np.int16)                         # the r < 3 tail: literals
    code = np.where((j >= full) & (r >= 3), np.where(j == full, 256 + r - 3, -1), code)
    code = np.where(j < full, np.where(j % MAX_MATCH == 0, 256 + MAX_MATCH - 3, -1), code)
    sym[idx] = code
    return sym


def symbol_starts(sym):
    return np.flatnonzero(sym >= 0)


# ----------------------------------------------------------------------------- window slides
def slide_pos(sym, k, w, rowlen):
    """Loop-top position (a symbol start, or n) at which zlib's window slides for the k-th time
    (k >= 1), or None.  fill_window runs at a loop top only when the lookahead is at most 258; the
    k-th slide needs strstart >= (k+1)w - 262 there.  The input is fed one filtered row at a time,
    so before the loop top at p the data read ends at the first row end beyond q + 258 (q: the
    previous symbol start), capped by the window at (k+1)w."""
    n = len(sym)
    cap = (k + 1) * w
    p = cap - 262
    if p > n:
        return None
    q = p - 1
    while q >= 0 and sym[q] < 0:
        q -= 1
    while p < n and sym[p] < 0:
        p += 1
    while True:
        if p >= n or p >= cap - MAX_MATCH:
            return p
        e = min((((q + MAX_MATCH) // rowlen) + 1) * rowlen, n)
        if min(e, cap) - p <= MAX_MATCH:
            return p
        q = p
        p += 1
        while p < n and sym[p] < 0:
            p += 1


def stored_ok(sym, bstart, bend, last, w, rowlen):
    """zlib passes a buffer to the stored-block check only while block_start >= 0: the block's first
    byte minus w for every slide before its flush (loop tops before bend; for the final block, at
    or before n)."""
    n = len(sym)
    lim = n + 1 if last else bend
    j_max = (lim - 1 + 262) // w - 1
    if j_max <= 0:
        return True
    count = j_max - 1
    p = slide_pos(sym, j_max, w, rowlen)
    if p is not None and p < lim:
        count += 1
    return bstart >= count * w


# ----------------------------------------------------------------------------- trees
def _smaller(freq, depth, n, m):
    return freq[n] < freq[m] or (freq[n] == freq[m] and depth[n] <= depth[m])


def _downheap(heap, heap_len, freq, depth, k):
    v = heap[k]
    j = k << 1
    while j <= heap_len:
        if j < heap_len and _smaller(freq, depth, heap[j + 1], heap[j]):
            j += 1
        if _smaller(freq, depth, v, heap[j]):
            break
        heap[k] = heap[j]
        k = j
        j <<= 1
    heap[k] = v


def build_tree(freq_in, elems, slen, extra, base, max_length, acc):
    """trees.c build_tree + gen_bitlen + gen_codes for one tree.  acc: [opt_len, static_len],
    updated in place.  Returns (lens[elems], codes[elems], max_code)."""
    freq = [0] * HEAP_SIZE
    freq[:elems] = list(freq_in)
    depth = [0] * HEAP_SIZE
    dad = [0] * HEAP_SIZE
    ln = [0] * HEAP_SIZE
    heap = [0] * (HEAP_SIZE + 1)
    heap_len, heap_max, max_code = 0, HEAP_SIZE, -1
    for n in range(elems):
        if freq[n]:
            heap_len += 1
            heap[heap_len] = max_code = n
    while heap_len < 2:
        if max_code < 2:
            max_code += 1
            node = max_code
        else:
            node = 0
        heap_len += 1
        heap[heap_len] = node
        freq[node] = 1
        depth[node] = 0
        acc[0] -= 1
        if slen is not None:
            acc[1] -= slen[node]
    for n in range(heap_len // 2, 0, -1):
        _downheap(heap, heap_len, freq, depth, n)
    node = elems
    while True:
        n = heap[1]
        heap[1] = heap[heap_len]
        heap_len -= 1
        _downheap(heap, heap_len, freq, depth, 1)
        m = heap[1]
        heap_max -= 1
        heap[heap_max] = n
        heap_max -= 1
        heap[heap_max] = m
        freq[node] = freq[n] + freq[m]
        depth[node] = max(depth[n], depth[m]) + 1
        dad[n] = dad[m] = node
        heap[1] = node
        node += 1
        _downheap(heap, heap_len, freq, depth, 1)
        if heap_len < 2:
            break
    heap_max -= 1
    heap[heap_max] = heap[1]
    # gen_bitlen
    bl_count = [0] * 16
    ln[heap[heap_max]] = 0
    overflow = 0
    for h in range(heap_max + 1, HEAP_SIZE):
        n = heap[h]
        bits = ln[dad[n]] + 1
        if bits > max_length:
            bits, overflow = max_length, overflow + 1
        ln[n] = bits
        if n > max_code:
            continue
        bl_count[bits] += 1
        xbits = extra[n - base] if n >= base else 0
        acc[0] += freq[n] * (bits + xbits)
        if slen is not None:
            acc[1] += freq[n] * (slen[n] + xbits)
    if overflow:
        while True:
            bits = max_length - 1
            while bl_count[bits] == 0:
                bits -= 1
            bl_count[bits] -= 1
            bl_count[bits + 1] += 2
            bl_count[max_length] -= 1
            overflow -= 2
            if overflow <= 0:
                break
        h = HEAP_SIZE
        for bits in range(max_length, 0, -1):
            n = bl_count[bits]
            while n:
                h -= 1
                m = heap[h]
                if m > max_code:
                    continue
                if ln[m] != bits:
                    acc[0] += (bits - ln[m]) * freq[m]
                    ln[m] = bits
                n -= 1
    lens = [ln[n] if n <= max_code and freq[n] else 0 for n in range(elems)]
    return lens, gen_codes(lens, max_code), max_code


def _scan_runs(lens, max_code):
    """The (symbol, extra value, extra bits) sequence scan_tree counts and send_tree sends."""
    out = []
    prevlen, nextlen, count = -1, lens[0], 0
    max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
    for n in range(max_code + 1):
        curlen = nextlen
        nextlen = lens[n + 1] if n + 1 <= max_code else 0xFFFF
        count += 1
        if count < max_count and curlen == nextlen:
            continue
        if count < min_count:
            out += [(curlen, 0, 0)] * count
        elif curlen != 0:
            if curlen != prevlen:
                out.append((curlen, 0, 0))
                count -= 1
            out.append((16, count - 3, 2))
        elif count <= 10:
            out.append((17, count - 3, 3))
        else:
            out.append((18, count - 11, 7))
        count, prevlen = 0, curlen
        if nextlen == 0:
            max_count, min_count = 138, 3
        elif curlen == nextlen:
            max_count, min_count = 6, 3
        else:
            max_count, min_count = 7, 4
    return out


class Block:
    """One deflate block: its symbol range, trees, type and bits."""


def block_trees(lfreq, dfreq, stored_len, can_store):
    """trees.c _tr_flush_block's decision for one block's frequencies (END_BLOCK counted)."""
    acc = [0, 0]
    llen, lcode, lmax = build_tree(lfreq, L_CODES, STATIC_LLEN, EXTRA_LBITS, 257, 15, acc)
    dlen, dcode, dmax = build_tree(dfreq, D_CODES, STATIC_DLEN, EXTRA_DBITS, 0, 15, acc)
    runs = _scan_runs(llen, lmax) + _scan_runs(dlen, dmax)
    blfreq = [0] * BL_CODES
    for sym, _, _ in runs:
        blfreq[sym] += 1
    blacc = [0, 0]
    bllen, blcode, _ = build_tree(blfreq, BL_CODES, None, EXTRA_BLBITS, 0, 7, blacc)
    acc[0] += blacc[0]
    max_blindex = BL_CODES - 1
    while max_blindex >= 3 and bllen[BL_ORDER[max_blindex]] == 0:
        max_blindex -= 1
    acc[0] += 3 * (max_blindex + 1) + 5 + 5 + 4
    opt_lenb = (acc[0] + 3 + 7) >> 3
    static_lenb = (acc[1] + 3 + 7) >> 3
    if static_lenb <= opt_lenb:
        opt_lenb = static_lenb
    b = Block()
    b.opt_len, b.static_len = acc
    if stored_len + 4 <= opt_lenb and can_store:
        b.type = STORED
    elif static_lenb == opt_lenb:
        b.type = STATIC
        llen, lcode, dlen, dcode = STATIC_LLEN[:L_CODES], STATIC_LCODE[:L_CODES], STATIC_DLEN, \
            STATIC_DCODE
    else:
        b.type = DYNAMIC
        hdr = [(lmax + 1 - 257, 5), (dmax + 1 - 1, 5), (max_blindex + 1 - 4, 4)]
        hdr += [(bllen[BL_ORDER[r]], 3) for r in range(max_blindex + 1)]
        for sym, xv, xb in runs:
            hdr.append((blcode[sym], bllen[sym]))
            if xb:
                hdr.append((xv, xb))
        b.hdr = hdr
    b.llen, b.lcode, b.dlen, b.dcode = llen, lcode, dlen, dcode
    return b


# ----------------------------------------------------------------------------- bit writer
class BitWriter:
    """LSB-first bit writer over numpy pieces (each piece: values, bit counts)."""

    def __init__(self):
        self.vals, self.nbits, self.bits = [], [], 0

    def put(self, vals, nbits):
        vals = np.atleast_1d(np.asarray(vals, dtype=np.uint64))
        nbits = np.atleast_1d(np.asarray(nbits, dtype=np.int64))
        keep = nbits > 0
        self.vals.append(vals[keep])
        self.nbits.append(nbits[keep])
        self.bits += int(nbits.sum())

    def align(self):
        pad = -self.bits % 8
        if pad:
            self.put([0], [pad])

    def tobytes(self):
        v = np.concatenate(self.vals) if self.vals else np.zeros(0, np.uint64)
        nb = np.concatenate(self.nbits) if self.nbits else np.zeros(0, np.int64)
        total = int(nb.sum())
        out = np.zeros(-(-total // 8), dtype=np.uint8)
        step = 1 << 22
        starts = np.concatenate([[0], np.cumsum(nb)[:-1]]).astype(np.int64)
        for a in range(0, len(v), step):
            vv, bb, ss = v[a:a + step], nb[a:a + step], starts[a:a + step]
            owner = np.repeat(np.arange(len(vv)), bb)
            pos = np.arange(int(bb.sum()), dtype=np.int64) + (ss[0] if len(ss) else 0)
            within = pos - ss[owner]
            bits = ((vv[owner] >> within.astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
            np.bitwise_or.at(out, pos >> 3, (bits << (pos & 7).astype(np.uint8)).astype(np.uint8))
        return out.tobytes()


# ----------------------------------------------------------------------------- the encoder
class Encoded:
    """encode()'s result: the file and the intermediates the device also reports."""


def deflate(stream, rowlen):
    """The raw deflate stream of zlib level 1 / Z_RLE over `stream`, plus its blocks."""
    s = np.asarray(stream, dtype=np.uint8)
    n = len(s)
    _, zbits = window_bits(n)
    w = 1 << zbits
    sym = parse(s)
    pos = symbol_starts(sym)
    nsym = len(pos)
    nblocks = nsym // SYMS_PER_BLOCK + 1
    bw = BitWriter()
    blocks = []
    for k in range(nblocks):
        last = k == nblocks - 1
        a, z = k * SYMS_PER_BLOCK, min((k + 1) * SYMS_PER_BLOCK, nsym)
        bstart = int(pos[a]) if a < nsym else n
        bend = int(pos[z]) if z < nsym else n
        codes = sym[pos[a:z]].astype(np.int64)
        is_match = codes >= 256
        lc = np.where(is_match, codes - 256, 0)
        lsym = np.where(is_match, 257 + LENGTH_CODE[lc], codes)
        lfreq = np.bincount(lsym, minlength=L_CODES)
        lfreq[END_BLOCK] += 1
        dfreq = np.zeros(D_CODES, dtype=np.int64)
        dfreq[0] = int(is_match.sum())
        b = block_trees([int(x) for x in lfreq], [int(x) for x in dfreq], bend - bstart,
                        stored_ok(sym, bstart, bend, last, w, rowlen))
        b.start, b.end, b.nsym, b.bit_start = bstart, bend, z - a, bw.bits
        bw.put([(b.type << 1) | int(last)], [3])
        if b.type == STORED:
            assert bend - bstart <= 0xFFFF
            bw.align()
            ln = bend - bstart
            bw.put([ln & 0xFFFF, ~ln & 0xFFFF], [16, 16])
            bw.put(s[bstart:bend], np.full(ln, 8))
        else:
            if b.type == DYNAMIC:
                v, nb = zip(*b.hdr)
                bw.put(v, nb)
            lcode, llen = np.array(b.lcode, np.uint64), np.array(b.llen, np.int64)
            xb = np.where(is_match, LENGTH_XBITS[lc], 0)
            xv = np.where(is_match, LENGTH_XVAL[lc], 0).astype(np.uint64)
            db = np.where(is_match, b.dlen[0], 0)
            dv = np.full(len(codes), b.dcode[0], np.uint64)
            # one symbol = code | extra << len | distance code << (len + extra)
            sl = llen[lsym]
            val = lcode[lsym] | (xv << sl.astype(np.uint64)) | \
                (dv << (sl + xb).astype(np.uint64))
            bw.put(np.where(is_match, val, lcode[lsym]), sl + xb + db)
            bw.put([b.lcode[END_BLOCK]], [b.llen[END_BLOCK]])
        b.bits = bw.bits - b.bit_start
        blocks.append(b)
    bw.align()
    return bw.tobytes(), sym, nsym, blocks


def encode(img):
    """uint8 [H, W, 3] RGB -> (PNG bytes equal to cv2.imencode('.png', img[..., ::-1]), Encoded)."""
    img = np.asarray(img)
    H, W, _ = img.shape
    stream = filter_rows(img)
    body, sym, nsym, blocks = deflate(stream, 3 * W + 1)
    z = zlib_header(len(stream)) + body + struct.pack(">I", adler32(stream))
    out = bytearray(b"\x89PNG\r\n\x1a\n" + ihdr(H, W))
    for c in range(0, len(z), IDAT_BYTES):
        out += chunk(b"IDAT", z[c:c + IDAT_BYTES])
    out += chunk(b"IEND", b"")
    e = Encoded()
    e.stream, e.sym, e.nsym, e.blocks, e.body, e.zstream = stream, sym, nsym, blocks, body, z
    return bytes(out), e
