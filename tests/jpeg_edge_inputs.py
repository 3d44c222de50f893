"""JPEG files built from chosen quantised coefficients, at the edges where a decoder that matches
cv2.imdecode on encoder-written files can still differ from it: IDCT arithmetic past the range an
encoder writes from [0, 255] pixels, 16-bit quantisers, colour and upsampling extremes, DC
prediction sums, and entropy-code corners.

`baseline` writes a sequential (SOF0) file from coefficients in decode order (the layout of
jpeg_oracle.coefficients, DC after the prediction) under any sampling, 8- or 16-bit DQT, Huffman
tables optimised for the data (T.81 K.2) and a restart interval.  Each builder returns `Case`s,
each of which states counts of the edge it was built for (`census` keys, see
test_jpeg_edge_oracle.py, which recomputes them from the file).  `progressive` re-encodes a
builder's files under two of jpeg_reencode's scan scripts.
"""
from __future__ import annotations

import dataclasses
import struct

import numpy as np

import jpeg_reencode as JR
from jpeg_reencode import _optimal_table, _Writer
from matterport_maskrcnn_with_tensorflow_serving_b200 import jpeg as J

ZZ = [int(v) for v in J.ZIGZAG[:64]]          # natural index of zig-zag position k
GRAY = [(1, 1)]
SAMPLINGS = {"444": [(1, 1)] * 3, "422": [(2, 1), (1, 1), (1, 1)],
             "420": [(2, 2), (1, 1), (1, 1)], "440": [(1, 2), (1, 1), (1, 1)],
             "411": [(4, 1), (1, 1), (1, 1)]}
# cv2's (libjpeg's jcparam.c) quality tables, natural order, from the T.81 Annex K tables
_K1 = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
                14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
                18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
_K2 = np.array([17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32)


def quality_table(q, chroma=False):
    """jcparam.c jpeg_quality_scaling + jpeg_add_quant_table (baseline clamp to [1, 255])."""
    s = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip(((_K2 if chroma else _K1) * s + 50) // 100, 1, 255).astype(np.int64)


@dataclasses.dataclass
class Case:
    name: str
    blob: bytes
    counts: dict                 # census key -> the count of that edge in the file
    refused: bool = False        # jpeg.parse / Plan raises, or the device reports a status
    cv2_decodes: bool = False    # a refused file cv2.imdecode still decodes (DESIGN §3.20)


def _seg(code, payload):
    return b"\xff" + bytes([code]) + struct.pack(">H", len(payload) + 2) + payload


def geometry(samp, W, H):
    """(mcux, mcuy, blocks per MCU) of a sequential scan: a one-component scan is not
    interleaved, its MCU is one block."""
    if len(samp) == 1:
        return -(-W // 8), -(-H // 8), 1
    hmax, vmax = max(h for h, _ in samp), max(v for _, v in samp)
    return -(-W // (8 * hmax)), -(-H // (8 * vmax)), sum(h * v for h, v in samp)


def from_grids(grids, samp, W, H):
    """Per-component block grids int64 [rows, cols, 64] (at least the MCU-padded size) -> the
    decode-order layout [MCUs * blocks per MCU, 64]."""
    mcux, mcuy, bpm = geometry(samp, W, H)
    out = np.zeros((mcuy, mcux, bpm, 64), dtype=np.int64)
    if len(samp) == 1:
        out[:, :, 0] = grids[0][:mcuy, :mcux]
        return out.reshape(-1, 64)
    c0 = 0
    for g, (h, v) in zip(grids, samp):
        for dy in range(v):
            for dx in range(h):
                out[:, :, c0 + dy * h + dx] = g[dy:mcuy * v:v, dx:mcux * h:h][:mcuy, :mcux]
        c0 += h * v
    return out.reshape(-1, 64)


def grid_shape(samp, W, H, ci):
    """(rows, cols) of component ci's MCU-padded block grid."""
    mcux, mcuy, _ = geometry(samp, W, H)
    if len(samp) == 1:
        return mcuy, mcux
    h, v = samp[ci]
    return mcuy * v, mcux * h


def _dc_event(diff):
    n = abs(int(diff)).bit_length()
    return n, (diff if diff >= 0 else diff - 1) & ((1 << n) - 1), n


def ac_events(blk):
    """jchuff.c's AC symbols of one block: [(symbol, extra bits value, extra bit count)]."""
    ev, r = [], 0
    for k in range(1, 64):
        v = int(blk[ZZ[k]])
        if v == 0:
            r += 1
            continue
        while r > 15:
            ev.append((0xF0, 0, 0))
            r -= 16
        n = abs(v).bit_length()
        ev.append(((r << 4) | n, (v if v >= 0 else v - 1) & ((1 << n) - 1), n))
        r = 0
    if r:
        ev.append((0x00, 0, 0))
    return ev


def baseline(coef, quant, samp, W, H, ri=0, dqt16=False, raw_ac=None, raw_dc=None, fill=0,
             tables=None):
    """A sequential baseline file: SOI, JFIF, DQT (one table per component, 16-bit entries when
    `dqt16` or an entry exceeds 255), SOF0, DHT (luma slot 0, chroma slot 1), DRI, SOS, data, EOI.
    `coef` int64 [MCUs * bpm, 64] natural order with absolute DC values (diffs are taken per
    component, reset at each restart); `raw_ac` / `raw_dc` map a block index to its own AC events
    or DC event (symbol, bits, n); `fill` 0xFF bytes go before each RSTn and before EOI; `tables`
    maps ("dc" | "ac", slot) to a (bits, vals) table used in place of the optimal one."""
    raw_ac, raw_dc, tables = raw_ac or {}, raw_dc or {}, tables or {}
    mcux, mcuy, bpm = geometry(samp, W, H)
    mcus = mcux * mcuy
    assert coef.shape == (mcus * bpm, 64), (coef.shape, mcus, bpm)
    comp_of = [0] if len(samp) == 1 else [ci for ci, (h, v) in enumerate(samp)
                                          for _ in range(h * v)]
    slot = [0 if ci == 0 else 1 for ci in range(len(samp))]
    ev = []                      # ("dc" | "ac", slot, symbol, bits, n) and ("rst", k)
    last = [0] * len(samp)
    for m in range(mcus):
        if ri and m and m % ri == 0:
            ev.append(("rst", m // ri - 1))
            last = [0] * len(samp)
        for c in range(bpm):
            b = m * bpm + c
            ci = comp_of[c]
            diff = int(coef[b, 0]) - last[ci]
            last[ci] = int(coef[b, 0])
            ev.append(("dc", slot[ci]) + (raw_dc[b] if b in raw_dc else _dc_event(diff)))
            ev += [("ac", slot[ci]) + e for e in (raw_ac[b] if b in raw_ac else ac_events(coef[b]))]
    head = bytearray(b"\xff\xd8") + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for ci, q in enumerate(quant):
        q = np.asarray(q, dtype=np.int64)
        assert q.min() >= 1 and q.max() <= 65535
        wide = dqt16 or q.max() > 255
        head += _seg(0xDB, bytes([(0x10 if wide else 0) | ci]) +
                     q[ZZ].astype(">u2" if wide else np.uint8).tobytes())
    comps = b"".join(bytes([ci + 1, (1 << 4 | 1) if len(samp) == 1 else (h << 4 | v), ci])
                     for ci, (h, v) in enumerate(samp))
    head += _seg(0xC0, struct.pack(">BHHB", 8, H, W, len(samp)) + comps)
    codes = {}
    dht = b""
    for kind, tc in (("dc", 0), ("ac", 1)):
        for s in sorted(set(slot)):
            if (kind, s) in tables:
                bits, vals = tables[(kind, s)]
            else:
                freq = [0] * 256
                for e in ev:
                    if e[0] == kind and e[1] == s:
                        freq[e[2]] += 1
                bits, vals = _optimal_table(freq)
            codes[(kind, s)] = JR._codes(bits, vals)
            dht += bytes([tc << 4 | s]) + bytes(bits) + bytes(vals)
    head += _seg(0xC4, dht)
    if ri:
        head += _seg(0xDD, struct.pack(">H", ri))
    head += _seg(0xDA, bytes([len(samp)]) + b"".join(
        bytes([ci + 1, slot[ci] << 4 | slot[ci]]) for ci in range(len(samp))) + b"\x00\x3f\x00")
    w = _Writer()
    for e in ev:
        if e[0] == "rst":
            w.flush()
            w.out += b"\xff" * fill + bytes([0xFF, 0xD0 + (e[1] & 7)])
            continue
        code, n = codes[(e[0], e[1])][e[2]]
        w.bits(code, n)
        w.bits(e[3], e[4])
    w.flush()
    return bytes(head) + bytes(w.out) + b"\xff" * fill + b"\xff\xd9"


def _q(v, n=3):
    return [np.full(64, v, dtype=np.int64) for _ in range(n)]


def _one(samp, W, H, fill_blocks, quant, name, counts, **kw):
    """A file whose blocks come from fill_blocks(component, grid rows, grid cols) -> grid."""
    grids = [fill_blocks(ci, *grid_shape(samp, W, H, ci)) for ci in range(len(samp))]
    return Case(name, baseline(from_grids(grids, samp, W, H), quant, samp, W, H, **kw), counts)


# ---------------------------------------------------------------------------------------- IDCT
def idct_dc(rng):
    """Dequantised DC at +-8191, +-8192, +-8193 in DC-only blocks (the pass-1 shortcut's << 2
    wraps past 8191), reached with quantiser 1 and with large quantisers."""
    vals = [8191, 8192, 8193, -8191, -8192, -8193]
    out = []
    for qdc, div in ((1, 1), (8191, None), (4096, None)):
        blocks = []
        for v in vals:
            if div is None and v % qdc:
                continue
            blocks.append(v // (div or qdc))
        q = np.ones(64, dtype=np.int64)
        q[0] = qdc
        W = 8 * len(blocks)
        coef = np.zeros((len(blocks), 64), dtype=np.int64)
        coef[:, 0] = blocks
        dq = {v: sum(1 for b in blocks if b * qdc == v) for v in vals}
        out.append(Case(f"idct_dc_q{qdc}", baseline(coef, [q], GRAY, W, 8),
                        {f"dc_dq_{v}": n for v, n in dq.items()}))
    return out


def idct_sums(rng):
    """The 16-bit sums in0 + in4, in0 - in4, in7 + in3 and in5 + in1 of pass 1 at 32767 / -32768
    (inside int16) and at 32768 / -32769 (wrapping), one column each, quantiser 1."""
    pairs = {(0, 4, 1): [(16383, 16384), (16384, 16384), (-16384, -16384), (-16384, -16385)],
             (0, 4, -1): [(16383, -16384), (16384, -16384), (-16384, 16384), (-16385, 16384)],
             (7, 3, 1): [(16383, 16384), (16384, 16384), (-16384, -16384), (-16385, -16384)],
             (5, 1, 1): [(16384, 16383), (16384, 16384), (-16384, -16384), (-16384, -16385)]}
    blocks = []
    for (a, b, _), vs in pairs.items():
        blk = np.zeros((8, 8), dtype=np.int64)
        for col, (va, vb) in enumerate(vs):
            blk[a, col], blk[b, col] = va, vb
        blocks.append(blk.reshape(64))
    coef = np.stack(blocks)
    return [Case("idct_sums", baseline(coef, _q(1, 1), GRAY, 8 * len(blocks), 8),
                 {"sum_inside": 8, "sum_wraps": 8})]


def idct_pass1(rng):
    """Pass-1 outputs just inside and just past int16 (packssdw saturates them): in0 and in2 of
    one column, whose row-0 output is about 4 in0 + 5.23 in2."""
    blocks = []
    for in0, in2 in ((6000, 1600), (6000, 1790), (-6000, -1600), (-6000, -1790)):
        blk = np.zeros((8, 8), dtype=np.int64)
        blk[0, 0], blk[2, 0] = in0, in2
        blocks.append(blk.reshape(64))
    # rows 0 and 7 of each column: 32362 / 33361 and their negatives
    return [Case("idct_pass1", baseline(np.stack(blocks), _q(1, 1), GRAY, 32, 8),
                 {"p1_near": 4, "p1_over": 4})]


def idct_pass2(rng):
    """Pass-2 outputs where jidctint.c's x & 1023 table and the SIMD saturation disagree
    from DC-only blocks below the shortcut's wrap.  A DC-only block's pass-2 output is
    (dq * 4 * 8192 + 2^17) >> 18 in all 64 pixels: 4100 -> 513, 8191 -> 1024, -4108 -> -513 and
    -8191 -> -1024 disagree; 2047, 4000, -4000 and -4100 (-> -512) do not."""
    dcs = [2047, 4000, 4100, 8191, -4000, -4100, -4108, -8191]
    coef = np.zeros((len(dcs), 64), dtype=np.int64)
    coef[:, 0] = dcs
    return [Case("idct_pass2", baseline(coef, _q(1, 1), GRAY, 8 * len(dcs), 8),
                 {"p2_disagree": 4 * 64})]


def idct_wrap_zero(rng):
    """Rows 1-7 nonzero in the raw coefficients, zero once dequantised (coef * q = 65536): the
    shortcut is decided on the raw values, so the full path runs and saturates."""
    blocks = []
    for dc in (8192, 8191, -8193):
        blk = np.zeros(64, dtype=np.int64)
        blk[0], blk[8] = dc, 2            # row 1, column 0
        blocks.append(blk)
    q = np.ones(64, dtype=np.int64)
    q[8] = 32768
    return [Case("idct_wrap_zero", baseline(np.stack(blocks), [q], GRAY, 24, 8),
                 {"wrap_zero": 3, "q_32768": 1})]


def idct_row0(rng):
    """Blocks whose nonzero coefficients are all in row 0 (the shortcut's domain with AC)."""
    coef = np.zeros((16, 64), dtype=np.int64)
    coef[:, :8] = rng.integers(-2000, 2001, (16, 8))
    coef[:8, 0] = [8191, 8192, -8192, -8193, 4096, 100, 0, 1]
    coef[15, 0] = 0
    n = int((coef[:, 1:8] != 0).any(axis=1).sum())
    return [Case("idct_row0", baseline(coef, _q(1, 1), GRAY, 128, 8), {"row0_ac": n})]


def idct_big_quant(rng):
    """16-bit quantisers of 32767, 32768 and 65535 (signed 16-bit: 32767, -32768, -1), under
    random small coefficients."""
    out = []
    for qv in (32767, 32768, 65535):
        q = np.full(64, qv, dtype=np.int64)
        q[::3] = rng.integers(1, 65536, 22)
        coef = rng.integers(-3, 4, (64, 64)) * (rng.random((64, 64)) < 0.3)
        out.append(Case(f"idct_quant_{qv}", baseline(coef, [q], GRAY, 64, 64),
                        {f"q_{qv}": int((q == qv).sum())}))
    return out


def idct_random_ac(rng):
    """Spec-conforming baseline data (|AC| <= 1023) under cv2's quality 10, 50 and 90 tables:
    every AC coefficient uniform in [-20, 20], or in [-1023, 1023] in a sparse tenth of the
    positions; 4:2:0 and gray."""
    out = []
    for q in (10, 50, 90):
        for samp, W, H in ((GRAY, 64, 64), (SAMPLINGS["420"], 48, 40)):
            mcux, mcuy, bpm = geometry(samp, W, H)
            n = mcux * mcuy * bpm
            coef = rng.integers(-20, 21, (n, 64))
            sparse = rng.random((n, 64)) < 0.1
            coef[sparse] = rng.integers(-1023, 1024, int(sparse.sum()))
            coef[:, 0] = rng.integers(-60, 61, n)
            quant = [quality_table(q, ci > 0) for ci in range(len(samp))]
            out.append(Case(f"idct_random_q{q}_{'gray' if len(samp) == 1 else '420'}",
                            baseline(coef, quant, samp, W, H), {"conforming_blocks": n}))
    return out


# ----------------------------------------------------------------------- colour and upsampling
def colour_dc_grid(pairs, samp_name="444"):
    """A DC-only 4:4:4 file (quantiser 8: sample = 128 + DC / 8 exactly) with one 8x8 block per
    (y, cb, cr) triple of `pairs`, laid out on a square-ish grid."""
    n = len(pairs)
    cols = int(np.ceil(np.sqrt(n)))
    rows = -(-n // cols)
    samp = SAMPLINGS[samp_name]
    grids = []
    for ci in range(3):
        g = np.zeros((rows, cols, 64), dtype=np.int64)
        g[:, :, 0].reshape(-1)[:n] = (np.asarray([p[ci] for p in pairs]) - 128)
        grids.append(g)
    coef = from_grids(grids, samp, 8 * cols, 8 * rows)
    return baseline(coef, _q(8), samp, 8 * cols, 8 * rows)


def colour_grids(step=1):
    """(Y, Cr) with Cb = 128, (Y, Cb) with Cr = 128, and (Cb, Cr) with Y = 128: every pair at
    step 1 (three 2048 x 2048 files), or every `step`-th value."""
    v = range(0, 256, step)
    grids = {"y_cr": [(y, 128, c) for y in v for c in v],
             "y_cb": [(y, c, 128) for y in v for c in v],
             "cb_cr": [(128, b, c) for b in v for c in v]}
    return [Case(f"colour_{k}_step{step}", colour_dc_grid(p), {"dc_pairs": len(p)})
            for k, p in grids.items()]


def checkerboards(rng):
    """0 / 255 block checkerboards (DC-only blocks, dequantised DC +-1024) under all five
    samplings and gray, at odd sizes, so every upsampler meets full-swing steps at its edges."""
    out = []
    for name, samp in [("gray", GRAY)] + list(SAMPLINGS.items()):
        for W, H in ((37, 23), (17, 9)):
            def fill(ci, r, c, samp=samp):
                g = np.zeros((r, c, 64), dtype=np.int64)
                sign = np.where((np.arange(r)[:, None] + np.arange(c)[None, :] + ci) % 2, 1, -1)
                g[:, :, 0] = 128 * sign          # quantiser 8: +-1024, the 0 / 255 extremes
                return g
            out.append(_one(samp, W, H, fill, _q(8, len(samp)), f"checker_{name}_{W}x{H}",
                            {"checker_blocks": sum(int(np.prod(grid_shape(samp, W, H, ci)))
                                                   for ci in range(len(samp)))}))
    return out


def narrow_chroma(rng):
    """Chroma 1, 2 and 3 samples wide (and tall): jdsample.c switches from replication to fancy
    upsampling at 3 (the image is 2, 4 and 6 pixels wide in 4:2:0 and 4:2:2)."""
    out = []
    for name in ("420", "422"):
        samp = SAMPLINGS[name]
        for W in (1, 2, 3, 4, 5, 6):
            H = W + 1

            def fill(ci, r, c):
                return rng.integers(-300, 301, (r, c, 64)) * (rng.random((r, c, 64)) < 0.4)
            cw = -(-W // 2)
            out.append(_one(samp, W, H, fill, _q(2), f"narrow_{name}_{W}x{H}",
                            {f"chroma_w{cw}": 1}))
    return out


# ------------------------------------------------------------------------------------------ DC
def dc_edges(rng):
    """DC prediction sums that cross int16 (JCOEF stores them truncated: the device must too),
    DC categories 12 to 15, a sum that crosses int32 (the device refuses it, cv2 need not) and a
    DC symbol of 16 (both refuse it)."""
    out = []
    # 40 blocks: running DC climbs by 30000 per block past 2^15 and on to ~1.2e6
    n = 40
    coef = np.zeros((n, 64), dtype=np.int64)
    coef[:, 0] = np.arange(1, n + 1) * 30000
    coef[:, 1] = 1
    cross = int(((coef[:, 0] < -32768) | (coef[:, 0] > 32767)).sum())
    out.append(Case("dc_int16_cross", baseline(coef, _q(1, 1), GRAY, 8 * n, 8),
                    {"dc_outside_int16": cross}))
    # categories 12 .. 15 up and down
    dcs = []
    for cat in range(12, 16):
        dcs += [(1 << (cat - 1)), -(1 << (cat - 1))]
    coef = np.zeros((len(dcs), 64), dtype=np.int64)
    coef[:, 0] = np.cumsum(np.asarray(dcs))
    cats = {f"dc_cat_{c}": 2 for c in range(12, 16)}
    out.append(Case("dc_categories", baseline(coef, _q(1, 1), GRAY, 8 * len(dcs), 8), cats))
    # a sum past int32: 65 538 category-15 diffs of 32767 (a 2048 x 2056 gray image).  The
    # device refuses it; libjpeg-turbo checks only in decode_mcu_slow, which it uses in the last
    # ~512 bytes of the data, so cv2 decodes this file (the sum wraps, the stored int16 agrees)
    W, H = 8 * 256, 8 * 257
    nb = (W // 8) * (H // 8)
    coef = np.zeros((nb, 64), dtype=np.int64)
    coef[:, 0] = np.arange(1, nb + 1, dtype=np.int64) * 32767
    out.append(Case("dc_int32_overflow", baseline(coef, _q(1, 1), GRAY, W, H),
                    {"dc_int32_refused": 1}, refused=True, cv2_decodes=True))
    # DC symbol 16 (no extra bits are defined for it)
    coef = np.zeros((4, 64), dtype=np.int64)
    out.append(Case("dc_symbol_16", baseline(coef, _q(1, 1), GRAY, 32, 8,
                                             raw_dc={2: (16, 0, 0)}),
                    {"dc_symbol_16": 1}, refused=True))
    return out


# ------------------------------------------------------------------------------ entropy decode
def entropy_edges(rng):
    """AC categories 11 to 15, codes of 16 bits (past the 9-bit fast table), one-code tables,
    all-EOB blocks, ZRL runs ending at index 63 and runs past it (the guard entries), restart
    interval 1 and fill bytes before RSTn and EOI."""
    out = []
    # AC categories 11-15
    coef = np.zeros((10, 64), dtype=np.int64)
    for i, cat in enumerate(range(11, 16)):
        coef[2 * i, ZZ[1 + i]] = (1 << cat) - 1
        coef[2 * i + 1, ZZ[60 - i]] = -(1 << (cat - 1))
    out.append(Case("ac_categories", baseline(coef, _q(1, 1), GRAY, 80, 8),
                    {f"ac_cat_{c}": 2 for c in range(11, 16)}))
    # codes of 10 to 16 bits (past the 9-bit fast lookup): an AC table with one code of each
    # length 2 .. 15 and three of 16 bits, over EOB, runs 0-14 of value +-1 and value +-2
    alphabet = [0x00] + [(r << 4) | 1 for r in range(15)] + [0x02]
    bits = [0] + [1] * 14 + [3]
    raw, blk, k = {}, [], 1
    for sym in rng.choice(alphabet[1:], 2000).tolist():
        r, n = sym >> 4, sym & 15
        if k + r > 63:
            raw[len(raw)] = blk + ([(0x00, 0, 0)] if k <= 63 else [])
            blk, k = [], 1
        blk.append((sym, int(rng.integers(0, 1 << n)), n))
        k += r + 1
    raw[len(raw)] = blk + ([(0x00, 0, 0)] if k <= 63 else [])
    nb = len(raw)
    out.append(Case("long_codes", baseline(np.zeros((nb, 64), dtype=np.int64), _q(1, 1), GRAY,
                                           8 * nb, 8, raw_ac=raw,
                                           tables={("ac", 0): (bits, alphabet)}),
                    {"ac_code_len_16": 1}))
    # one-code tables: all-EOB blocks with equal DC (DC table: symbol 0 only, AC: EOB only)
    coef = np.zeros((33, 64), dtype=np.int64)
    coef[:, 0] = 5
    out.append(Case("all_eob_one_code", baseline(coef, _q(3, 1), GRAY, 8 * 11, 24),
                    {"eob_blocks": 33}))
    # ZRL runs ending at index 63 (the block's end, no EOB), and runs that go past it
    coef = np.zeros((6, 64), dtype=np.int64)
    coef[2, ZZ[63]] = 7                       # three ZRLs, then run 14 to k = 63
    raw = {0: [(0xF0, 0, 0)] * 2 + [(0xE2, 3, 2), (0xF0, 0, 0)],      # value at k = 47, ZRL
           1: [(0x01, 0, 1), (0xD1, 1, 1)] + [(0xF0, 0, 0)] * 3,     # k = 1, k = 15, 3 ZRLs
           3: [(0xF0, 0, 0)] * 3 + [(0xF1, 1, 1)],                   # k = 49 + 15 = 64
           4: [(0x21, 1, 1)] + [(0xF0, 0, 0)] * 3 + [(0xF2, 3, 2)],   # k = 52 + 15 = 67
           5: [(0xF0, 0, 0)] * 4}                                    # the fourth ZRL: k = 64
    out.append(Case("zrl_runs", baseline(coef, _q(1, 1), GRAY, 48, 8, raw_ac=raw),
                    {"zrl_to_63": 2, "run_past_63": 3}))
    # restart interval 1, with and without fill bytes, 4:2:0
    samp = SAMPLINGS["420"]
    for fill in (0, 3):
        def f(ci, r, c):
            return rng.integers(-50, 51, (r, c, 64)) * (rng.random((r, c, 64)) < 0.3)
        out.append(_one(samp, 40, 24, f, _q(4), f"rst1_fill{fill}",
                        {"fill_bytes": 6 * fill, "restart_units": 6},
                        ri=1, fill=fill))
    # units of exactly k * 32 bits: a one-code DC table (a 1-bit code) and DC diffs of category
    # 15 (+-16384 after each restart's reset, then +-32767): 16 bits; one AC of +-4096 (category
    # 13, a 1-bit code) at index 1: 14 bits; EOB (a 2-bit code): 32 bits per block, restart
    # interval k
    for k in (1, 2, 32, 128):
        nb = 256
        coef = np.zeros((nb, 64), dtype=np.int64)
        j = np.arange(nb) % k                 # DC 16384, -16383, 16384, ... in each unit
        coef[:, 0] = np.where(j % 2, -16383, 16384) * rng.choice([-1, 1], nb // k).repeat(k)
        coef[:, 1] = 4096 * rng.choice([-1, 1], nb)
        out.append(Case(f"units_{32 * k}_bits",
                        baseline(coef, _q(1, 1), GRAY, 128, 128, ri=k,
                                 tables={("ac", 0): ([1, 1] + [0] * 14, [0x0D, 0x00])}),
                        {f"units_of_{32 * k}_bits": nb // k}))
    return out


def ff_boundaries(rng):
    """0xFF data bytes (stuffed as FF 00) at the byte offsets where subsequences of S bits begin,
    for S = 32 .. 4096: a gray file whose AC values are all 1023 (ten one bits each)."""
    out = []
    # each block: DC symbol 0 (optimal: a one-code table, 1 bit) then AC values chosen so the
    # extra bits are all ones: value 2^n - 1 codes as n one bits; many in a row make 0xFF bytes
    nb = 256
    coef = np.zeros((nb, 64), dtype=np.int64)
    coef[:, ZZ[1:61]] = 1023                 # category 10, extra bits 1111111111
    coef[:, 0] = 0
    out.append(Case("ff_runs", baseline(coef, _q(1, 1), GRAY, 8 * 16, 8 * 16),
                    {f"ff_at_S_{S}": 1 for S in (32, 64, 128, 256, 512, 1024, 2048, 4096)}))
    return out


def colour_pairs(rng):
    """The three DC-only colour grids at every 17th value (the full grids: colour_grids(1))."""
    return colour_grids(step=17)


BUILDERS = [idct_dc, idct_sums, idct_pass1, idct_pass2, idct_wrap_zero, idct_row0,
            idct_big_quant, idct_random_ac, checkerboards, narrow_chroma, dc_edges,
            entropy_edges, ff_boundaries, colour_pairs]

PROGRESSIVE_SCRIPTS = ("al4", "eob_whole")


def progressive(cases):
    """Each accepted case re-encoded under PROGRESSIVE_SCRIPTS (its coefficients, DC truncated
    to int16 as the baseline decode stores it)."""
    import jpeg_oracle as JO

    out = []
    for c in cases:
        if c.refused:
            continue
        dc = JO.coefficients(c.blob)[0][:, 0].astype(np.int64)
        for s in PROGRESSIVE_SCRIPTS:
            if s == "eob_whole" and np.ptp(dc) > 32767:
                continue      # its DC scan (Al = 0) could need a DC difference of category 16
            out.append(Case(f"{c.name}_prog_{s}", JR.reencode(c.blob, JR.SCRIPTS[s]), {}))
    return out


def all_cases(seed=0):
    rng = np.random.default_rng(seed)
    return [c for b in BUILDERS for c in b(rng)]
