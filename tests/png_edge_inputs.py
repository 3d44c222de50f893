"""PNG files whose deflate streams sit where the device PNG decoder (csrc/png_decode.cu) can part
from cv2.imdecode: streams zlib never writes.  A small deflate writer takes explicit tokens,
code lengths and code-length sequences; the builders put one-code and empty distance codes,
15-bit codes, code-length repeats across the literal/distance boundary, length 258 as 284 + 31,
distances at the window's far end under every CINFO, reaches to the stream's first byte,
stored blocks at every bit phase, dynamic blocks packed past the finder's slots and false block
headers in front of the decoder; besides, invalid streams before the last row and unfilter edges.

Each builder returns Cases that state counts of their edge (`census` keys).  `census` recomputes
those counts from the file's bytes with `walk`, a deflate decoder written for these tests that
records every block's header, code lengths, code-length sequence and tokens, and
`candidates`, the block-start finder's acceptance rules (zlib's inflate on a dynamic header)
restated for every bit of a stream."""
import dataclasses
import struct
import zlib

import numpy as np

import png_decode_inputs as P

LBASE, LEXT, DBASE, DEXT, ORDER = P.LBASE, P.LEXT, P.DBASE, P.DEXT, P.ORDER
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32
TILE_BITS = 1024                                 # mrx.h MRX_PNG_DEC_TILE_BITS
ST_CODE, ST_DIST = 4, 8                          # mrx.h MRX_PNG_ST_*


# ------------------------------------------------------------------ writer
class BitWriter:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):                         # LSB first
        self.acc |= v << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def code(self, c, n):                        # a Huffman code, MSB first
        self.put(int(format(c, f"0{n}b")[::-1], 2) if n else 0, n)

    def bit(self):
        return 8 * len(self.out) + self.n

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)

    def data(self):
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def codes(lengths):
    """[(code, length) or None] of the canonical code with these lengths."""
    count = [0] * 16
    for l in lengths:
        count[l] += 1
    count[0] = 0
    nxt, c = [0] * 16, 0
    for l in range(1, 16):
        c = (c + count[l - 1]) << 1
        nxt[l] = c
    out = []
    for l in lengths:
        out.append((nxt[l], l) if l else None)
        if l:
            nxt[l] += 1
    return out


def limited_lengths(freqs, limit=15):
    """Huffman code lengths of at most `limit` bits (package-merge); one used symbol gets 1."""
    used = sorted((f, s) for s, f in enumerate(freqs) if f)
    lens = [0] * len(freqs)
    if len(used) == 1:
        lens[used[0][1]] = 1
        return lens
    leaves = [(f, [s]) for f, s in used]
    cur = list(leaves)
    for _ in range(limit - 1):
        packs = [(cur[i][0] + cur[i + 1][0], cur[i][1] + cur[i + 1][1])
                 for i in range(0, len(cur) - 1, 2)]
        cur = sorted(leaves + packs, key=lambda x: x[0])
    for _, ss in cur[:2 * len(used) - 2]:
        for s in ss:
            lens[s] += 1
    return lens


def len_sym(length):
    return 285 if length == 258 else 257 + max(k for k in range(28) if LBASE[k] <= length)


def dist_sym(d):
    return max(k for k in range(30) if DBASE[k] <= d)


def match(length, dist, lsym=None):
    """A match token: ('m', length symbol, its extra, distance symbol, its extra)."""
    ls = len_sym(length) if lsym is None else lsym
    ds = dist_sym(dist)
    return ("m", ls, length - LBASE[ls - 257], ds, dist - DBASE[ds])


def tokens_for(raw, matches):
    """Literals of `raw`, but a match at each position of `matches` {pos: (length, dist[, lsym])}."""
    out, p = [], 0
    while p < len(raw):
        if p in matches:
            m = matches[p]
            out.append(match(*m))
            p += m[0]
        else:
            out.append(raw[p])
            p += 1
    return out


def copy_matches(raw, matches):
    """raw with each match's bytes copied from its source, in order (overlaps as inflate does)."""
    raw = bytearray(raw)
    for p in sorted(matches):
        length, dist = matches[p][:2]
        for k in range(length):
            raw[p + k] = raw[p + k - dist]
    return raw


def rle(lens, prev=None):
    """Code-length symbols [(sym, extra)] of `lens`; `prev` lets a 16 open the sequence."""
    out, i = [], 0
    while i < len(lens):
        v, j = lens[i], i
        while j < len(lens) and lens[j] == v:
            j += 1
        n = j - i
        if v == 0 and n >= 3:
            while n >= 11:
                k = min(n, 138)
                out.append((18, k - 11))
                n -= k
            if n >= 3:
                out.append((17, n - 3))
                n = 0
            out += [(0, 0)] * n
        else:
            if prev != v:
                out.append((v, 0))
                n -= 1
            while n >= 3:
                k = min(n, 6)
                out.append((16, k - 3))
                n -= k
            out += [(v, 0)] * n
        prev, i = v, j
    return out


def _body(w, tokens, lit, dist):
    for t in tokens:
        if isinstance(t, tuple):
            _, ls, le, ds, de = t
            w.code(*lit[ls])
            w.put(le, LEXT[ls - 257] if ls < 286 else 0)
            w.code(*dist[ds])
            w.put(de, DEXT[ds] if ds < 30 else 0)
        else:
            w.code(*lit[t])
    w.code(*lit[256])


def token_freqs(tokens):
    lf, df = [0] * 286, [0] * 30
    lf[256] = 1
    for t in tokens:
        if isinstance(t, tuple):
            lf[t[1]] += 1
            df[t[3]] += 1
        else:
            lf[t] += 1
    return lf, df


def dynamic(w, tokens, lit_lens=None, dist_lens=None, final=0, seq=None, cl_lens=None,
            hclen=None, joint=False, hlit=None, hdist=None, body=True):
    """A dynamic block.  Lengths default to limited Huffman codes of the tokens, trimmed to
    HLIT >= 257 / HDIST >= 1; `seq` ([(sym, extra)]) replaces the code-length run encoding (zlib's
    two runs, or one crossing run with `joint`); hlit/hdist/hclen override the header fields."""
    lf, df = token_freqs(tokens)
    if lit_lens is None:
        lit_lens = limited_lengths(lf)
        lit_lens = lit_lens[:max(257, max(s for s, l in enumerate(lit_lens) if l) + 1)]
    if dist_lens is None:
        dist_lens = limited_lengths(df) if any(df) else [0]
        dist_lens = dist_lens[:max([1] + [s + 1 for s, l in enumerate(dist_lens) if l])]
    if seq is None:
        seq = rle(list(lit_lens) + list(dist_lens)) if joint else rle(lit_lens) + rle(dist_lens)
    if cl_lens is None:
        cf = [0] * 19
        for s, _ in seq:
            cf[s] += 1
        if sum(1 for f in cf if f) == 1:
            cf[18 if cf[0] else 0] = 1                # a complete code needs two symbols
        cl_lens = limited_lengths(cf, 7)
    if hclen is None:
        hclen = max([4] + [k + 1 for k in range(19) if cl_lens[ORDER[k]]])
    w.put(final, 1)
    w.put(2, 2)
    w.put((hlit or len(lit_lens)) - 257, 5)
    w.put((hdist or len(dist_lens)) - 1, 5)
    w.put(hclen - 4, 4)
    for k in range(hclen):
        w.put(cl_lens[ORDER[k]], 3)
    cc = codes(cl_lens)
    for s, e in seq:
        w.code(*cc[s])
        w.put(e, {16: 2, 17: 3, 18: 7}.get(s, 0))
    if body:
        lit = codes(list(lit_lens) + [0] * (288 - len(lit_lens)))
        _body(w, tokens, lit, codes(list(dist_lens) + [0] * (32 - len(dist_lens))))


def fixed(w, tokens, final=0):
    w.put(final, 1)
    w.put(1, 2)
    _body(w, tokens, codes(FIXED_LIT), codes(FIXED_DIST))


def stored(w, data, final=0):
    w.put(final, 1)
    w.put(0, 2)
    w.align()
    w.put(len(data), 16)
    w.put(0xFFFF ^ len(data), 16)
    w.out += data


def zwrap(deflate, raw, cinfo=7):
    cmf = cinfo << 4 | 8
    flg = 31 - (cmf * 256) % 31
    return bytes([cmf, flg]) + deflate + struct.pack(">I", zlib.adler32(bytes(raw)))


# ------------------------------------------------------------------ images
def rows(rng, h, w, top=256):
    """Filtered bytes of an 8-bit gray h x w image, filter 0 on every row, data below `top`."""
    r = rng.integers(0, top, size=(h, w + 1), dtype=np.uint8)
    r[:, 0] = 0
    return bytearray(r.tobytes())


def gray_file(raw, h, w, z, split=None):
    blob = P.write(np.zeros((h, w, 1), np.uint8), 0, 8, stream=bytes(raw))
    return P.with_zlib_stream(blob, z, split)


def gray_pixels(raw, h, w):
    a = np.frombuffer(bytes(raw), np.uint8).reshape(h, w + 1)[:, 1:]
    return np.repeat(a[..., None], 3, -1)


@dataclasses.dataclass
class Case:
    name: str
    blob: bytes                    # the file, its stream in one IDAT chunk
    counts: dict                   # census key -> count of that edge in the file
    pixels: np.ndarray = None      # the intended image; None: refused
    status: int = 0                # the expected MRX_PNG_ST_* bit of a refused file
    cv2: tuple = (True, True, True)   # cv2 decodes it with IDAT whole, in 1- and 7-byte chunks
    stride: int = 0                # filtered row length (census of distance sources)
    raw: bytes = None              # the intended filtered stream


def _gray_case(name, raw, h, w, z, counts, **kw):
    return Case(name, gray_file(raw, h, w, z), counts, gray_pixels(raw, h, w), stride=w + 1,
                raw=bytes(raw), **kw)


def _refused(name, raw, h, w, z, counts, status, cv2=(False, False, False)):
    return Case(name, gray_file(raw, h, w, z), counts, None, status, cv2, w + 1, None)


# ------------------------------------------------------------------ builders
def distance_codes(rng):
    """One-code distance codes of length 1 (symbol 0, and symbol 5 alone), empty distance codes
    (HDIST 1 and 30), literal-only blocks; each after a first block, so the finder meets it."""
    h, w = 6, 40
    raw = rows(rng, h, w, 4)
    n = len(raw)
    m1 = {p: (4, 1) for p in range(50, 110, 8)}
    m5 = {p: (3, 7) for p in range(140, 200, 7)}
    raw = copy_matches(raw, {**m1, **m5})
    t1, t5 = tokens_for(raw[40:120], {p - 40: v for p, v in m1.items()}), \
        tokens_for(raw[120:200], {p - 120: v for p, v in m5.items()})
    bw = BitWriter()
    fixed(bw, list(raw[:40]))
    dynamic(bw, t1, dist_lens=[1])
    dynamic(bw, t5, dist_lens=[0] * 5 + [1])
    dynamic(bw, list(raw[200:230]), dist_lens=[0])
    dynamic(bw, list(raw[230:n]), dist_lens=[0] * 30, final=1)
    z = zwrap(bw.data(), raw)
    return [_gray_case("distance codes", raw, h, w, z,
                       {"dist_one_code": 2, "dist_empty": 2, "literal_only": 3, "hdist_1": 2,
                        "hdist_30": 1})]


def long_codes(rng):
    """Literal/length and distance codes of every length 11-15 (the slow path past the 10-bit
    lookup), and a literal/length code of 256 15-bit codes and seven short ones."""
    out = []
    # 16 symbols of lengths 1..15, 15: literals 0..11, length 257, literals 12, 13, end of block
    lit = [0] * 286
    for s, l in zip(list(range(12)) + [257, 12, 13, 256], list(range(1, 16)) + [15]):
        lit[s] = l
    dist = list(range(1, 16)) + [15] + [0] * 14
    h, w = 5, 700
    raw = rows(rng, h, w, 14)
    ms = {}
    for k in range(120):
        ds = k % 16
        d = DBASE[ds] + int(rng.integers(0, 1 << DEXT[ds]))
        r = 1 + k % (h - 1)
        p = r * (w + 1) + 1 + (k // 16) * 80 + ds * 4
        if p - d >= 0 and p + 3 < (r + 1) * (w + 1):
            ms[p] = (3, d)
    raw = copy_matches(raw, ms)
    bw = BitWriter()
    dynamic(bw, tokens_for(raw, ms), lit, dist, final=1)
    out.append(_gray_case("codes of 11-15 bits", raw, h, w, zwrap(bw.data(), raw),
                          {"lit_len_11": 1, "lit_len_12": 1, "lit_len_13": 1, "lit_len_14": 1,
                           "lit_len_15": 1, "dist_len_11": 1, "dist_len_12": 1,
                           "dist_len_13": 1, "dist_len_14": 1, "dist_len_15": 1,
                           "hclen_19": 1}))
    lit = [15] * 263 + [0] * 23
    for s in range(7):
        lit[s] = s + 1
    h, w = 8, 300
    raw = rows(rng, h, w)
    ms = {r * (w + 1) + 10 + 40 * k: (3 + k, 1 + k) for r in range(1, h) for k in range(6)}
    raw = copy_matches(raw, ms)
    bw = BitWriter()
    dynamic(bw, tokens_for(raw, ms), lit, [2, 2, 2, 3, 3], final=1)
    out.append(_gray_case("all 15-bit but seven", raw, h, w, zwrap(bw.data(), raw),
                          {"lit_all_15": 1, "lit_len_15": 1}))
    return out


def code_length_runs(rng):
    """Code-length sequences zlib never sends: a 16 and an 18 across the literal/distance
    boundary, 16 at the first distance entry, an 18 of 138, HCLEN 19 with trailing zeros, HLIT 257
    and 286, HDIST 1 and 30."""
    h, w = 4, 90
    raw = rows(rng, h, w, 8)
    ms = {20: (17, 3), 60: (25, 19), 200: (21, 40), 240: (30, 7)}
    raw = copy_matches(raw, ms)
    cut = [0, 120, 180, 300, len(raw)]
    seg = [tokens_for(raw[a:b], {p - a: m for p, m in ms.items() if a <= p < b})
           for a, b in zip(cut, cut[1:])]
    # 32 codes of 5 bits: literals 0..7, end of block, lengths 263..285; 28 distances of 5 bits
    # and two of 4: the 5s run from the literal/length lengths on into the distance lengths
    lit = [0] * 286
    for s in list(range(8)) + [256] + list(range(263, 286)):
        lit[s] = 5
    dist = [5] * 28 + [4, 4]
    bw = BitWriter()
    dynamic(bw, seg[0], lit, dist, joint=True)
    # HLIT 286 whose 29 length lengths are zero, then 20 zero distance lengths: an 18 across; the
    # 248 zeros of literals 8..255 hold an 18 of 138
    lit2 = [0] * 286
    for s, l in zip(list(range(8)) + [256], [3, 3, 3, 3, 3, 3, 3, 4, 4]):
        lit2[s] = l
    dynamic(bw, seg[1], lit2, [0] * 20 + [1, 1], joint=True)
    # the distance lengths opened by a 16 that repeats the last literal/length length
    dynamic(bw, seg[2], lit, dist, seq=rle(lit) + rle(dist, prev=lit[-1]))
    # HLIT 257, HDIST 1 (no distance code), HCLEN 19 though 15, 1 and 14 have no length
    dynamic(bw, seg[3], lit2[:257], [0], hclen=19, final=1)
    z = zwrap(bw.data(), raw)
    return [_gray_case("code-length runs", raw, h, w, z,
                       {"cl_cross": 2, "cl16_first_dist": 1, "cl18_138": 2, "hclen_19": 1,
                        "hlit_257": 1, "hlit_286": 3, "hdist_30": 2, "hdist_1": 1,
                        "dist_empty": 1})]


def lengths(rng):
    """Every length code at its base and its base + the largest extra, and 258 as 284 + 31 and as
    285, in a dynamic and in a fixed block: copies at distance 1 of an all-zero image."""
    want = []
    for ls in range(257, 286):
        want += [(LBASE[ls - 257], ls), (LBASE[ls - 257] + (1 << LEXT[ls - 257]) - 1, ls)]
    want += [(258, 284)] * 3 + [(258, 285)] * 3
    total = 1 + sum(l for l, _ in want)
    w = 199
    h = -(-(2 * total) // (w + 1))
    raw = bytearray(h * (w + 1))
    out = []
    bw = BitWriter()
    toks = [0] + [match(l, 1, ls) for l, ls in want]
    dynamic(bw, toks)
    toks2 = [match(l, 1, ls) for l, ls in want]
    rest = len(raw) - 2 * total + 1
    fixed(bw, toks2 + [0] * rest, final=1)
    out.append(_gray_case("lengths", raw, h, w, zwrap(bw.data(), raw),
                          {"len284_31": 6, "len285_258": 6, "len_base": 29, "len_top": 29}))
    return out


# cv2 4.13 (libpng 1.6) on window + 1 under CINFO 0..6, the source in the copy's row and in an
# earlier row: it decodes with the stream in one IDAT chunk, never in 1-byte chunks, and in 7-byte
# chunks as the chunk boundaries fall (the device refuses them all)
T, F = True, False
CV2_WINDOW_PLUS_1 = [((T, F, T), (T, F, T)), ((T, F, F), (T, F, T)), ((T, F, F), (T, F, F)),
                     ((T, F, F), (T, F, T)), ((T, F, T), (T, F, T)), ((T, F, F), (T, F, F)),
                     ((T, F, T), (T, F, F))]


def distances(rng):
    """Distances 1, 32 506, 32 507-32 768; window and window + 1 under every CINFO, with the
    source in the copy's own row and in an earlier row; 1 500 under CINFO 2 in one row."""
    out = []

    def one(name, d, same_row, cinfo, length=5, counts=None, refused=False, cv2=None):
        w = d + length + 30 if same_row else 97
        h = 2 if same_row else -(-(d + 200) // (w + 1)) + 1
        raw = rows(rng, h, w)
        if same_row:
            p = (h - 1) * (w + 1) + 1 + d + 10
        else:
            p = (h - 1) * (w + 1) + 30
        ms = {p: (length, d)}
        raw = copy_matches(raw, ms)
        bw = BitWriter()
        dynamic(bw, tokens_for(raw, ms), final=1)
        z = zwrap(bw.data(), raw, cinfo)
        key = {"dist_" + ("same_row" if same_row else "earlier_row"): 1}
        key.update(counts or {})
        if refused:
            out.append(_refused(name, raw, h, w, z, key, ST_DIST, cv2))
        else:
            out.append(_gray_case(name, raw, h, w, z, key))

    one("distance 1", 1, True, 7, 200, {"dist_1": 1})
    for d in (32506, 32507, 32508, 32640, 32767, 32768):
        one(f"distance {d}", d, d % 2 == 0, 7,
            counts={"dist_32506" if d == 32506 else "dist_far_end": 1})
    for cinfo in range(8):
        win = 256 << cinfo
        for same in (True, False):
            one(f"CINFO {cinfo} window, {'same' if same else 'earlier'} row", win, same, cinfo,
                counts={"dist_window": 1, f"cinfo_{cinfo}": 1})
            if win < 32768:
                one(f"CINFO {cinfo} window + 1, {'same' if same else 'earlier'} row", win + 1,
                    same, cinfo, counts={"dist_window_plus_1": 1, f"cinfo_{cinfo}": 1},
                    refused=True, cv2=CV2_WINDOW_PLUS_1[cinfo][not same])
    one("distance 1500 under CINFO 2 in one row", 1500, True, 2,
        counts={"dist_past_window": 1, "cinfo_2": 1}, refused=True, cv2=(True, False, False))
    return out


def reaches(rng):
    """A non-first dynamic block whose copy reaches exactly to the stream's first byte, and one
    that reaches one byte before it: the chain re-measures the block a candidate measured."""
    out = []
    h, w = 3, 50
    for past in (0, 1):
        raw = rows(rng, h, w, 16)
        first = 60
        p = first + 7
        d = p + past
        ms = {p: (9, d)}
        if not past:
            raw = copy_matches(raw, ms)
        bw = BitWriter()
        fixed(bw, list(raw[:first]))
        dynamic(bw, tokens_for(raw[first:], {k - first: v for k, v in ms.items()}), final=1)
        z = zwrap(bw.data(), raw)
        if past:
            out.append(_refused("reach one byte before the stream", raw, h, w, z,
                                {"reach_past": 1}, ST_DIST))
        else:
            out.append(_gray_case("reach to the stream's first byte", raw, h, w, z,
                                  {"reach_exact": 1}))
    return out


def stored_blocks(rng):
    """Stored blocks of 0, 1 and 65 535 bytes with their headers at all eight bit phases (a fixed
    block before each sets the phase), stored after a dynamic block, data across IDAT chunks."""
    out = []
    for big in (False, True):
        sizes = (65535,) if big else (0, 1)
        n_st = 8 * len(sizes)
        need = 8 * 80 + sum(sizes) * 8 + 400
        w = 255
        h = -(-need // (w + 1))
        raw = rows(rng, h, w, 144)
        bw = BitWriter()
        at = 0
        dynamic(bw, list(raw[:30]))
        at = 30
        stored(bw, bytes(raw[at:at + 5]))
        at += 5
        for phase in range(8):
            for size in sizes:
                j = (phase - (bw.bit() + 16) - 2) % 8        # 9-bit literals move the phase
                chunk = bytearray(raw[at:at + 40])
                hi = [k for k in range(40) if (at + k) % (w + 1)][:j]
                for k in hi:
                    chunk[k] = 144 + int(rng.integers(0, 112))
                raw[at:at + 40] = chunk
                fixed(bw, list(chunk))
                at += 40
                stored(bw, bytes(raw[at:at + size]))
                at += size
        fixed(bw, list(raw[at:]), final=1)
        counts = {f"stored_phase_{k}": len(sizes) for k in range(8)}
        counts.update({f"stored_len_{s}": 8 for s in sizes})
        counts.update({"stored_after_fixed": n_st, "stored_after_dynamic": 1})
        out.append(_gray_case(f"stored blocks of {sizes}", raw, h, w, zwrap(bw.data(), raw),
                              counts))
    return out


MIN_DYNAMIC_BITS = 100


def finder(rng):
    """Dynamic blocks of one literal each, ten or more per 1024-bit tile (past 1 and 4 slots);
    stored data made of valid dynamic blocks at every bit offset (false candidates); a false
    header whose block has no end-of-block code before the stream ends."""
    out = []
    h, w = 2, 40
    raw = rows(rng, h, w, 3)
    bw = BitWriter()
    for p in range(len(raw)):
        dynamic(bw, [raw[p]], final=int(p == len(raw) - 1))
    out.append(_gray_case("one literal per dynamic block", raw, h, w, zwrap(bw.data(), raw),
                          {"dense_tiles": 1}))
    # false candidates: a minimal dynamic block's bits at every bit offset inside stored data
    one = BitWriter()
    dynamic(one, [1, 2, 1], final=1)
    pb, nb = one.data(), one.bit()
    pay = BitWriter()
    for k in range(48):
        pay.put(int.from_bytes(pb, "little") & ((1 << nb) - 1), nb)
        pay.put(0, 1 + k % 8)
    pay.align()
    body = pay.data()
    w = len(body)
    h = 3
    raw = bytearray()
    for r in range(h):
        raw += b"\x00" + body
    bw = BitWriter()
    stored(bw, bytes(raw[:w + 1]))
    fixed(bw, list(raw[w + 1:w + 9]))
    stored(bw, bytes(raw[w + 9:2 * w + 2]))
    dynamic(bw, list(raw[2 * w + 2:]), final=1)
    out.append(_gray_case("false dynamic headers in stored data", raw, h, w,
                          zwrap(bw.data(), raw), {"false_candidates": 90}))
    # a false header with the end-of-block code 15 ones long, then zeros: its measure decodes
    # literal 0 bit after bit to the end of the stream
    lit = [0] * 257
    for s, l in zip(list(range(14)) + [14, 256], list(range(1, 15)) + [15, 15]):
        lit[s] = l
    fb = BitWriter()
    dynamic(fb, [], lit, [0], body=False, final=1)
    false_hdr = fb.data()
    w = 300
    raw = bytearray(w + 1)
    raw[1:1 + len(false_hdr)] = false_hdr
    bw = BitWriter()
    stored(bw, bytes(raw), final=1)
    out.append(_gray_case("false header measured to the stream's end", raw, 1, w,
                          zwrap(bw.data(), raw), {"false_to_end": 1}))
    return out


def _bad(name, write, counts, rng):
    """A stream refused before its last row: rows, a stored block of its first row, then the
    invalid block `write` draws."""
    h, w = 4, 30
    raw = rows(rng, h, w)
    bw = BitWriter()
    stored(bw, bytes(raw[:w + 1]))
    write(bw, raw[w + 1:])
    bw.put(0, 64)
    return _refused(name, raw, h, w, zwrap(bw.data(), raw), counts, ST_CODE)


def invalid(rng):
    """Streams zlib refuses, each in the block after the first row."""
    def hdr(hlit, hdist):
        return lambda bw, r: dynamic(bw, list(r), hlit=hlit, hdist=hdist)

    def cl(cl_lens, seq=None, lit=None, dist=None):
        return lambda bw, r: dynamic(bw, [], lit, dist, seq=seq, cl_lens=cl_lens, body=False)

    lit_ok = [8] * 256 + [8]
    lit_ok[0] = 0
    base = [8] * 255 + [0, 8]                 # 256 codes of 8 bits: complete
    cases = [
        ("HLIT 287", hdr(287, 1), {"hlit_287": 1}),
        ("HLIT 288", hdr(288, 1), {"hlit_288": 1}),
        ("HDIST 31", hdr(None, 31), {"hdist_31": 1}),
        ("HDIST 32", hdr(None, 32), {"hdist_32": 1}),
        ("incomplete code-length code", cl([0] * 8 + [1] + [0] * 10, []), {"cl_incomplete": 1}),
        ("empty code-length code", cl([0] * 19, [], [8] * 257, [1]), {"cl_empty": 1}),
        ("16 as the first code length", cl(None, [(16, 0)] + rle(base) + [(0, 0)], base, [0]),
         {"cl16_first": 1}),
        ("repeat past HLIT + HDIST", cl(None, rle(base) + [(17, 2)], base, [0]),
         {"cl_overrun": 1}),
        ("no end-of-block length", cl(None, rle([8] * 256 + [0]) + [(1, 0)], [8] * 256 + [0],
                                      [1]), {"error: invalid code -- missing end-of-block": 1}),
        ("HCLEN 4", lambda bw, r: dynamic(bw, [], [0] * 257, [0], seq=[(18, 127), (18, 108)],
                                          cl_lens=[1] + [0] * 17 + [1], hclen=4, body=False),
         {"hclen_4": 1}),
        ("over-subscribed literal/length code",
         cl(None, None, [1, 1] + [0] * 254 + [1], [1]), {"lit_over": 1}),
        ("incomplete literal/length code", cl(None, None, [2, 2] + [0] * 254 + [2], [1]),
         {"lit_incomplete": 1}),
        ("one 2-bit distance code", cl(None, None, base, [2]), {"dist_incomplete": 1}),
        ("over-subscribed distance code", cl(None, None, base, [1, 1, 1]), {"dist_over": 1}),
    ]
    out = [_bad(n, f, c, rng) for n, f, c in cases]
    for sym in (286, 287):
        out.append(_bad(f"fixed code {sym}", lambda bw, r, s=sym: fixed(
            bw, [r[0], ("m", s, 0, 0, 0)]), {f"fixed_{sym}": 1}, rng))
    for ds in (30, 31):
        out.append(_bad(f"distance code {ds}", lambda bw, r, d=ds: fixed(
            bw, [r[0], r[1], ("m", 257, 0, d, 0)]), {f"dist_code_{ds}": 1}, rng))
    return out


def pixels(rng):
    """Unfilter edges: Paeth's tie classes, Adam7 passes of more than 256 rows and of one
    column, rows of one byte under filters 1, 3 and 4 (zlib streams: the edge is the filter)."""
    out = []
    a = rng.integers(0, 5, size=(40, 61, 3), dtype=np.uint8)
    ties = {"paeth_ab": 100, "paeth_ac": 100, "paeth_bc": 100, "paeth_all": 100}
    out.append(Case("Paeth ties", P.write(a, 2, 8, filters=(4,)), ties, a,
                    raw=P.filtered_stream(a, 2, 8, 0, (4,))))
    g = rng.integers(0, 2, size=(24, 33, 1), dtype=np.uint8) * 255
    out.append(Case("Paeth ties, gray", P.write(g, 0, 8, filters=(4, 4, 1)), {},
                    np.repeat(g, 3, -1), raw=P.filtered_stream(g, 0, 8, 0, (4, 4, 1))))
    a = rng.integers(0, 256, size=(2100, 5, 3), dtype=np.uint8)
    out.append(Case("Adam7 of 2100 rows", P.write(a, 2, 8, interlace=1, filters=(4, 1, 3, 2)),
                    {"adam7_rows_gt256": 7}, a))
    a = rng.integers(0, 256, size=(300, 1, 1), dtype=np.uint8)
    out.append(Case("Adam7 of one column", P.write(a, 0, 8, interlace=1, filters=(1, 3, 4)),
                    {"adam7_one_col": 4}, np.repeat(a, 3, -1)))
    for f in (1, 3, 4):
        a = rng.integers(0, 256, size=(9, 1, 1), dtype=np.uint8)
        out.append(Case(f"one-byte rows, filter {f}", P.write(a, 0, 8, filters=(f,)),
                        {f"row_1byte_f{f}": 9}, np.repeat(a, 3, -1),
                        raw=P.filtered_stream(a, 0, 8, 0, (f,))))
        b = rng.integers(0, 2, size=(9, 5, 1), dtype=np.uint8)
        out.append(Case(f"one-byte rows of 1 bit, filter {f}", P.write(b, 0, 1, filters=(f,)),
                        {f"row_1byte_f{f}": 9}, np.repeat(b * 255, 3, -1)))
    return out


BUILDERS = [distance_codes, long_codes, code_length_runs, lengths, distances, reaches,
            stored_blocks, finder, invalid, pixels]


def all_cases(seed=0):
    return [c for b in BUILDERS for c in b(np.random.default_rng(seed))]


# ------------------------------------------------------------------ walker
class _Reader:
    def __init__(self, z, bit):
        self.z, self.pos = z, bit

    def get(self, n):
        v = 0
        for k in range(n):
            i = self.pos + k
            if i >> 3 < len(self.z):
                v |= ((self.z[i >> 3] >> (i & 7)) & 1) << k
        self.pos += n
        return v

    def over(self):
        return self.pos > 8 * len(self.z)


class Bad(Exception):
    pass


def _table(lens, kind):
    """{(length, code): symbol}, or Bad as inftrees.c: over-subscribed, or incomplete but for
    one code of length 1 (literal/length, distance) or for none (the code-length code too)."""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    left = 1
    for l in range(1, 16):
        left = 2 * left - count[l]
        if left < 0:
            raise Bad(f"invalid {kind} set")
    if left > 0 and sum(count) > 0 and (kind == "code lengths" or max(lens) != 1):
        raise Bad(f"invalid {kind} set")
    out, t = {}, codes(lens)
    for s, c in enumerate(t):
        if c:
            out[(c[1], c[0])] = s
    return out


def _sym(r, table, kind):
    code = 0
    for l in range(1, 16):
        code = code << 1 | r.get(1)
        if (l, code) in table:
            return table[(l, code)], l
    raise Bad(f"invalid {kind} code")


def header(r):
    """A dynamic block's header from after BTYPE: (record, literal/length and distance tables)."""
    hlit, hdist, hclen = r.get(5) + 257, r.get(5) + 1, r.get(4) + 4
    rec = {"hlit": hlit, "hdist": hdist, "hclen": hclen, "seq": []}
    try:
        return _header(r, rec)
    except Bad as e:
        raise Bad(e.args[0], rec)


def _header(r, rec):
    hlit, hdist, hclen = rec["hlit"], rec["hdist"], rec["hclen"]
    if hlit > 286 or hdist > 30:
        raise Bad("too many length or distance symbols", rec)
    cl = [0] * 19
    for k in range(hclen):
        cl[ORDER[k]] = r.get(3)
    rec["cl"] = cl
    if sum(1 for v in cl if v) == 0:
        raise Bad("invalid code lengths set")
    ct = _table(cl, "code lengths")
    lens = []
    while len(lens) < hlit + hdist:
        s, _ = _sym(r, ct, "code lengths")
        at = len(lens)
        if s < 16:
            lens.append(s)
            rec["seq"].append((s, 0, at))
            continue
        if s == 16:
            if not lens:
                rec["seq"].append((16, 0, 0))
                raise Bad("invalid bit length repeat")
            e = r.get(2)
            v, n = lens[-1], 3 + e
        else:
            e = r.get(3) if s == 17 else r.get(7)
            v, n = 0, (3 if s == 17 else 11) + e
        rec["seq"].append((s, e, at))
        if at + n > hlit + hdist:
            raise Bad("invalid bit length repeat")
        lens += [v] * n
    rec["lit"], rec["dist"] = lens[:hlit], lens[hlit:]
    if lens[256] == 0:
        raise Bad("invalid code -- missing end-of-block")
    lt = _table(rec["lit"], "literal/lengths")
    dt = _table(rec["dist"], "distances")
    return rec, lt, dt


def block(z, bit, out, wsize=1 << 15, base=None):
    """Decode the block at `bit` appending to bytearray `out`.  base=None: distances may reach
    before the stream's first byte, recorded (a candidate's measure).  Returns the record."""
    r = _Reader(z, bit)
    rec = {"bit": bit, "out": len(out), "final": r.get(1), "type": r.get(2), "tokens": [],
           "need": 0}
    try:
        if rec["type"] == 3:
            raise Bad("invalid block type")
        if rec["type"] == 0:
            r.pos = (r.pos + 7) & ~7
            n, nn = r.get(16), r.get(16)
            if n != 0xFFFF ^ nn:
                raise Bad("invalid stored block lengths")
            rec["len"] = n
            if r.pos // 8 + n > len(z):
                raise Bad("truncated")
            out += z[r.pos // 8:r.pos // 8 + n]
            r.pos += 8 * n
            rec["end"] = r.pos
            return rec
        if rec["type"] == 1:
            lt, dt = _table(FIXED_LIT, "literal/lengths"), _table(FIXED_DIST, "distances")
        else:
            h, lt, dt = header(r)
            rec.update(h)
        start = len(out)
        while True:
            s, l = _sym(r, lt, "literal/length")
            if r.over():
                raise Bad("truncated")
            if s < 256:
                out.append(s)
                rec["tokens"].append((s, l))
                continue
            if s == 256:
                break
            if s > 285:
                rec["bad_sym"] = s
                raise Bad("invalid literal/length code")
            e = r.get(LEXT[s - 257])
            d, dl = _sym(r, dt, "distance")
            if d > 29:
                rec["bad_sym"] = 1000 + d
                raise Bad("invalid distance code")
            de = r.get(DEXT[d])
            length, dist = LBASE[s - 257] + e, DBASE[d] + de
            if r.over():
                raise Bad("truncated")
            rec["tokens"].append((s, l, e, d, dl, de, length, dist, len(out)))
            if dist > wsize or (base is not None and dist > len(out)):
                raise Bad("invalid distance too far back")
            rec["need"] = max(rec["need"], dist - (len(out) - start))
            for _ in range(length):
                out.append(out[-dist] if dist <= len(out) else 0)
        rec["end"] = r.pos
        return rec
    except Bad as e:
        rec["error"] = e.args[0]
        if len(e.args) > 1:
            rec.update(e.args[1])
        rec["end"] = r.pos
        return rec


def walk(z):
    """(the stream's bytes, its block records; the last has 'error' when the stream is invalid)."""
    wsize = 256 << (z[0] >> 4)
    out, blocks, bit = bytearray(), [], 16
    while True:
        rec = block(z, bit, out, wsize, base=0)
        blocks.append(rec)
        if "error" in rec or rec["final"]:
            return bytes(out), blocks
        bit = rec["end"]


def candidates(z):
    """Every bit of z (from its third byte) where a dynamic block header starts that inflate
    accepts and that ends inside z."""
    out = []
    zz = bytes(z) + bytes(4)
    for i in range(2, len(z)):
        v = int.from_bytes(zz[i:i + 3], "little")
        for s in range(8):
            x = v >> s
            if (x >> 1) & 3 != 2 or (x >> 3) & 31 > 29 or (x >> 8) & 31 > 29:
                continue
            r = _Reader(z, 8 * i + s + 3)
            try:
                header(r)
            except Bad:
                continue
            if not r.over():
                out.append(8 * i + s)
    return out


def paeth_ties(raw, bpp, width_bytes):
    """Counts of Paeth's tie classes over the filter-4 bytes of a stream of rows."""
    stride = width_bytes + 1
    cnt = {"paeth_ab": 0, "paeth_ac": 0, "paeth_bc": 0, "paeth_all": 0}
    prev = bytes(width_bytes)
    for r in range(len(raw) // stride):
        f = raw[r * stride]
        line = bytearray(raw[r * stride + 1:(r + 1) * stride])
        for i in range(width_bytes):
            a = line[i - bpp] if i >= bpp else 0
            b = prev[i]
            c = prev[i - bpp] if i >= bpp else 0
            if f == 4:
                p = a + b - c
                pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                if pa == pb == pc:
                    cnt["paeth_all"] += 1
                elif pa == pb < pc:
                    cnt["paeth_ab"] += 1
                elif pa == pc < pb:
                    cnt["paeth_ac"] += 1
                elif pb == pc < pa:
                    cnt["paeth_bc"] += 1
            pred = (0, a, b, (a + b) // 2, P._paeth(a, b, c))[f]
            line[i] = (line[i] + pred) & 255
        prev = bytes(line)
    return cnt


def census(case):
    """The counts of every edge key in the case's file, from its bytes."""
    blob = case.blob
    ihdr = struct.unpack(">IIBBBBB", blob[16:29])
    w, h, depth, ct, _, _, il = ihdr
    z = P.zlib_stream(blob)
    _, blocks = walk(z)
    c = {}

    def add(k, n=1):
        c[k] = c.get(k, 0) + n

    win = 256 << (z[0] >> 4)
    add(f"cinfo_{z[0] >> 4}")
    prev_type = None
    seen_base, seen_top = set(), set()
    for k, b in enumerate(blocks):
        if b["type"] == 0 and "len" in b:
            add(f"stored_phase_{b['bit'] % 8}")
            if b["len"] in (0, 1, 65535):
                add(f"stored_len_{b['len']}")
            if prev_type == 1:
                add("stored_after_fixed")
            if prev_type == 2:
                add("stored_after_dynamic")
        if b["type"] == 2 and "hlit" in b:
            add(f"hlit_{b['hlit']}")
            if "cl" in b and "error" in b:
                kraft = sum(2.0 ** -v for v in b["cl"] if v)
                add("cl_empty" if kraft == 0 else "cl_incomplete" if kraft < 1 else "cl_ok")
            for name, lens in (("lit", b.get("lit")), ("dist", b.get("dist"))):
                if lens and "error" in b:
                    kraft = sum(2.0 ** -v for v in lens if v)
                    add(f"{name}_over" if kraft > 1 else f"{name}_incomplete" if kraft < 1
                        and sorted(v for v in lens if v) != [1] and kraft > 0 else f"{name}_ok")
            add(f"hdist_{b['hdist']}")
            add(f"hclen_{b['hclen']}")
            for s, e, at in b["seq"]:
                n = 1 if s < 16 else 3 + e if s == 16 else 3 + e if s == 17 else 11 + e
                if at < b["hlit"] < at + n:
                    add("cl_cross")
                if s == 16 and at == b["hlit"]:
                    add("cl16_first_dist")
                if s == 16 and at == 0:
                    add("cl16_first")
                if s > 15 and at + n > b["hlit"] + b["hdist"]:
                    add("cl_overrun")
                if s == 18 and e == 127:
                    add("cl18_138")
            if "dist" in b:
                dl = b["dist"]
                if sorted(v for v in dl if v) == [1]:
                    add("dist_one_code")
                if not any(dl):
                    add("dist_empty")
                ll = b["lit"]
                if len(ll) >= 257 and sum(1 for v in ll if v == 15) >= 250 and \
                        sum(1 for v in ll if 0 < v < 15) <= 8:
                    add("lit_all_15")
        if b["type"] in (1, 2) and "error" not in b:
            if not any(len(t) > 2 for t in b["tokens"]):
                add("literal_only")
            ls, ds = set(), set()
            for t in b["tokens"]:
                ls.add(t[1])
                if len(t) > 2:
                    s, l, e, d, dl, de, length, dist, at = t
                    ds.add(dl)
                    if s == 284 and e == 31:
                        add("len284_31")
                    if s == 285:
                        add("len285_258")
                    if e == 0:
                        seen_base.add(s)
                    if e == (1 << LEXT[s - 257]) - 1:
                        seen_top.add(s)
                    add_dist(add, dist, at, case.stride, win, b, k)
            for l in range(11, 16):
                if l in ls:
                    add(f"lit_len_{l}")
                if l in ds:
                    add(f"dist_len_{l}")
        if "error" in b:
            add("error: " + b["error"])
            _census_error(add, b, k, case.stride, win)
        prev_type = b["type"]
    add("len_base", len(seen_base))
    add("len_top", len(seen_top))
    # the finder
    if len(z) < 20000:
        cand = candidates(z)
        true = {b["bit"] for b in blocks if b["type"] == 2}
        per = {}
        for b in true:
            per[b // TILE_BITS] = per.get(b // TILE_BITS, 0) + 1
        if per and max(per.values()) > 4:
            add("dense_tiles")
        false = [x for x in cand if x not in true]
        add("false_candidates", len(false))
        for x in false:
            m = block(z, x, bytearray(), win)
            if m.get("error") == "truncated":
                add("false_to_end")
    # pixels
    if il:
        for p, (x0, y0, dx, dy) in enumerate(P.ADAM7):
            pw, ph = -(-(w - x0) // dx) if w > x0 else 0, -(-(h - y0) // dy) if h > y0 else 0
            if pw and ph > 256:
                add("adam7_rows_gt256")
            if pw == 1 and ph:
                add("adam7_one_col")
    bits_pp = P.CHANNELS[ct] * depth
    rb = (w * bits_pp + 7) // 8
    if not il and rb == 1:
        raw = zlib.decompressobj().decompress(z)
        for r in range(h):
            add(f"row_1byte_f{raw[r * 2]}")
    if not il and case.raw is not None and any(case.raw[r * (rb + 1)] == 4 for r in range(h)):
        for k, v in paeth_ties(case.raw, max(1, bits_pp // 8), rb).items():
            add(k, v)
    return c


def add_dist(add, dist, at, stride, win, b, k):
    if dist == 1:
        add("dist_1")
    if dist == 32506:
        add("dist_32506")
    if 32507 <= dist <= 32768:
        add("dist_far_end")
    if dist == win:
        add("dist_window")
    if stride:
        add("dist_same_row" if at // stride == (at - dist) // stride else "dist_earlier_row")
    if k > 0 and b["type"] == 2 and dist == at:
        add("reach_exact")


def _census_error(add, b, k, stride, win):
    if b["error"] == "invalid distance too far back":
        tok = b["tokens"][-1]
        dist, at = tok[7], tok[8]
        if dist > win:
            add("dist_window_plus_1" if dist == win + 1 else "dist_past_window")
            add("dist_same_row" if stride and at // stride == (at - dist) // stride
                else "dist_earlier_row")
        elif dist == at + 1 and k > 0:
            add("reach_past")
    if "bad_sym" in b:
        s = b["bad_sym"]
        add(f"fixed_{s}" if s < 1000 else f"dist_code_{s - 1000}")
    if b.get("hclen") == 4 and b["type"] == 2:
        add("hclen_4")
    if b.get("hlit", 0) > 286 or b.get("hdist", 0) > 30:
        add(f"hlit_{b['hlit']}" if b["hlit"] > 286 else f"hdist_{b['hdist']}")
