"""RGB images whose PNG encoding (csrc/png.cu, tests/png_oracle.py) reaches the paths of zlib's
block coding that real images do not: the 15- and 7-bit length limits, heap and cost ties, the
dummy nodes, the largest tree descriptions, the device's tile and block seams, stored blocks at
every bit phase, IDAT chunk ends and the Adler-32 range.

Every image is written as its filtered stream (Sub filter, filter byte 1 at each row start) and
turned into pixels by `png_inputs.image_from_stream`.  Most are one row, so the stream is the
filter byte 1 and then any 3W bytes.  A stream with no byte equal to its predecessor is all
literals, so its positions are its symbols and a block is exactly 16 383 positions.

Each builder returns Cases that state counts of the edges they target (`census` keys), and
`census(encoded)` recomputes those counts from the oracle's blocks.  Edges no image can have are
named in the builder's docstring with the reason."""
import dataclasses
import random
from collections import Counter

import numpy as np

import png_inputs
import png_oracle as P

TILE, SYMS, MAX = P.TILE, P.SYMS_PER_BLOCK, P.MAX_MATCH
MOD = 65521


@dataclasses.dataclass
class Case:
    name: str
    img: np.ndarray
    counts: dict                   # census key -> least count of that edge in the image


# ------------------------------------------------------------------ streams
def ordered(counts, prev):
    """The values of `counts` ({value: count}) in an order with no value equal to the one before
    it (the first differs from `prev`): always the most numerous value allowed, ties to the
    smallest.  Asserts that the counts allow it."""
    left = dict(counts)
    out = []
    for _ in range(sum(left.values())):
        v = max((v for v in left if left[v] and v != prev), key=lambda v: (left[v], -v))
        out.append(v)
        left[v] -= 1
        prev = v
    return np.array(out, np.uint8)


def noise(rng, n, prev):
    """n random bytes, none equal to the one before it (the first differs from `prev`)."""
    out = rng.integers(0, 255, n).astype(np.int64)
    for i in range(n):
        p = prev if i == 0 else out[i - 1]
        if out[i] >= p:
            out[i] += 1        # uniform over the 255 values other than p
    return out.astype(np.uint8)


def row_image(stream):
    """The one-row image whose filtered stream is `stream` (stream[0] == 1, len = 3W + 1)."""
    s = np.asarray(stream, np.uint8)
    assert s[0] == 1 and len(s) % 3 == 1 and len(s) >= 7, len(s)
    return png_inputs.image_from_stream(s[1:], 1, (len(s) - 1) // 3)


def pad_row(rng, parts):
    """Concatenated stream parts, then 1..3 noise bytes so that the length is 3W + 1."""
    s = np.concatenate(parts)
    k = (1 - len(s)) % 3 or 3
    return np.concatenate([s, noise(rng, k, s[-1])])


def with_filter_byte(counts):
    """A block's literal counts as a stream starting with the filter byte 1 (counts[1] >= 1)."""
    c = dict(counts)
    assert c.get(1, 0) >= 1
    c[1] -= 1
    return np.concatenate([[1], ordered(c, 1)]).astype(np.uint8)


def chain(m):
    """m counts whose Huffman tree is a chain of depth m - 1: each count above the sum of all
    but the largest before it, so the newest internal node is always one of the two smallest."""
    w = [1, 1, 1]
    while len(w) < m:
        w.append(sum(w[:-1]) + 1)
    return w


def chain_block(m, fill):
    """Literal counts of one block: chain(m) less its first 1 (END_BLOCK is that leaf) on the
    values 1.., then `fill` values sharing the rest of a full 16 383-symbol block (none: only the
    chain)."""
    c = {1 + i: n for i, n in enumerate(chain(m)[1:])}
    rest = SYMS - sum(c.values())
    for j in range(fill):
        c[100 + j] = rest // fill + (j < rest % fill)
    return c


def _to_row(counts):
    """The counts with the largest raised by 0..2 so that they total 1 mod 3 (a final block's
    bytes that end a one-row stream); the largest count of a chain may grow."""
    c = dict(counts)
    c[max(c, key=c.get)] += (1 - sum(c.values())) % 3
    return c


# ------------------------------------------------------------------ builders
def literal_overflow(rng):
    """Literal/length trees deeper than 15 bits: chain-shaped histograms (chain_block) whose
    overflow is 2, 4, 6 and 8, in a first block, a middle block and final blocks, three of them
    full 16 383-symbol blocks.

    Overflow 1 and odd overflows cannot occur: gen_bitlen counts every node, leaf or internal,
    whose depth it clamps, and every node but the root has a sibling at its own depth, so the
    nodes deeper than 15 come in pairs."""
    out = []
    s = with_filter_byte(chain_block(20, 4))                       # overflow 2, full, first
    out.append(Case("lit overflow 2, first block",
                    row_image(pad_row(rng, [s, noise(rng, 50, s[-1])])),
                    {"lit_overflow_2": 1, "lit_overflow_first": 1, "lit_overflow_full": 1}))
    a = noise(rng, SYMS, 0)
    a[0] = 1
    b = ordered(chain_block(16, 2), a[-1])                          # overflow 4, full, middle
    out.append(Case("lit overflow 4, middle block",
                    row_image(pad_row(rng, [a, b, noise(rng, 40, b[-1])])),
                    {"lit_overflow_4": 1, "lit_overflow_middle": 1}))
    c = ordered(_to_row(chain_block(19, 0)), a[-1])                # overflow 6, final
    out.append(Case("lit overflow 6, final block", row_image(np.concatenate([a, c])),
                    {"lit_overflow_6": 1, "lit_overflow_final": 1}))
    d = with_filter_byte(_to_row(chain_block(20, 0)))               # overflow 8, one block
    out.append(Case("lit overflow 8, only block", row_image(d),
                    {"lit_overflow_8": 1, "lit_overflow_final": 1}))
    return out


def _lengths_design(order, k, runs, seed):
    """Code lengths for the literals 0..255 and END_BLOCK (256) whose code-length symbols have
    chain-like counts: chain(11)'s largest k counts on the lengths of `order`, the rest of the
    Kraft sum on the shortest lengths that leave room for the remaining entries, then the zero
    or equal-length `runs` ((length, count): sent as 17, 18 or 16) spliced between unequal
    neighbours; every other neighbour differs, so no other run code is sent.  END_BLOCK gets 14,
    byte 1 a nonzero length.  Every length is -log2 of its frequency (2^(14 - length) bytes of
    16 384), so zlib's Huffman lengths are these."""
    c = Counter()
    for v, n in zip(order, chain(11)[::-1][:k]):
        c[v] += n
    zeros = c.pop(0, 0)
    units = sum(n << (14 - v) for v, n in c.items())
    left = 257 - zeros - sum(c.values())
    while left:
        v = next(v for v in range(2, 15) if units + (1 << (14 - v)) + left - 1 <= 1 << 14)
        c[v] += 1
        units += 1 << (14 - v)
        left -= 1
    assert units == 1 << 14
    c[0] = zeros
    for v, n in runs:
        c[v] -= n
    r = random.Random(seed)
    tot = sum(c.values())
    for _ in range(500):
        cc = dict(c)
        cc[14] -= 1
        prev, seq = None, []
        for i in range(tot - 1):
            cands = [v for v in cc if cc[v] and v != prev and not (i == 1 and v == 0)
                     and not (i == tot - 2 and v == 14)]
            if not cands:
                break
            v = max(cands, key=lambda v: (cc[v], r.random()))
            seq.append(v)
            cc[v] -= 1
            prev = v
        else:
            seq.append(14)
            for v, n in runs:
                j = next(j for j in range(3, len(seq) - 1)
                         if seq[j - 1] not in (0, v) and seq[j] not in (0, v))
                seq[j:j] = [v] * n
            return seq
    raise AssertionError("no arrangement")


def bitlength_overflow(rng):
    """Bit-length trees deeper than 7 bits, overflow 2, 4 and 6: one full block of literals
    whose code lengths (_lengths_design) send code-length symbols with chain-like counts, then one
    more literal, the final block (one literal plus END_BLOCK).  These are also the widest tree
    descriptions the inputs reach (`hdr_bits_max`).

    The widest a description can be: HLIT/HDIST/HCLEN and 19 three-bit lengths are 71 bits; the
    distance tree here always sends two lengths (only distance code 0 is used, and a dummy node
    joins it, or two when no match is coded); the literal tree at most 286.  Every code-length
    symbol is at most 7 bits, and a run code costs at most 7 + 7 bits for 11 or more entries or
    7 + 3 for 3 or more, never more than 7 bits an entry.  So a description is at most
    71 + 7 * 288 = 2 087 bits, inside the 2 560 bits (80 words) each block's table holds.

    A bit-length tree with a single used symbol cannot occur: the two distance lengths are 1, 1
    (symbol 1), and a literal tree of at least 257 entries holds a zero or a length other than 1."""
    out = []
    for name, order, runs, ovf in [
            ("bl overflow 2", (0, 14, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4), [], 2),
            ("bl overflow 4", (0, 14, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4), [(0, 11), (0, 3)], 4),
            ("bl overflow 6", (0, 14, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4),
             [(0, 11), (0, 3), (13, 4)], 6)]:
        lens = _lengths_design(order, 10, runs, 0)
        counts = {v: 1 << (14 - l) for v, l in enumerate(lens[:256]) if l}
        s = with_filter_byte(counts)
        out.append(Case(name, row_image(np.concatenate([s, noise(rng, 1, s[-1])])),
                        {f"bl_overflow_{ovf}": 1, "one_literal_eob": 1}))
    return out


def dummies(rng):
    """Trees with fewer than two codes: no match in a coded block (two dummy distance nodes),
    one distance code (one dummy), END_BLOCK alone in an empty final block (one dummy literal
    node), and one literal plus END_BLOCK (a final block of one symbol: a block of one literal
    value and more than three symbols holds a stretch, whose matches add length codes)."""
    f = np.array([1, 5, 9, 5, 9, 5, 9, 200, 9, 5] * 40, np.uint8)[:301]
    m = f.copy()
    m[40:60] = 9
    q = noise(rng, 3 * SYMS + 1, 0)                       # 49 150 symbols: 3 full blocks + EOB
    q[0] = 1
    return [Case("few values, no match", row_image(f), {"dist_empty": 1}),
            Case("few values, one run", row_image(m), {"dist_one": 1}),
            Case("3 x 16383 + 1 symbols", row_image(q), {"one_literal_eob": 1}),
            Case("16383 symbols", png_inputs.image_from_stream(
                png_inputs.run_free_stream(rng, 129, 42), 129, 42), {"eob_only": 1})]


# (seed, h, w, levels) of small random images found by searching with the oracle; see cost_ties
TIE_SEEDS = {"stored_tie": (12, 2, 11, 256), "stored_tie_m1": (32, 3, 8, 256),
             "stored_tie_p1": (11, 1, 7, 8), "static_tie": (233, 1, 5, 2),
             "static_tie_m1": (331, 1, 15, 8), "static_tie_p1": (172, 2, 8, 8)}


def _tie_image(seed, h, w, k):
    r = np.random.default_rng(seed)
    r.integers(1, 4), r.integers(2, 41), r.choice([2, 3, 4, 8, 256])   # the search's draws
    return (r.integers(0, k, (h, w, 3)) * (255 // max(k - 1, 1))).astype(np.uint8)


def cost_ties(rng):
    """Block-type decisions on a tie and one byte either side, in images of at most 3 x 40 found
    by a seeded search with the oracle: stored_len + 4 == opt_lenb (stored wins), == opt_lenb
    -+ 1; static_lenb == the dynamic length with stored losing (static wins), and -+ 1."""
    return [Case(f"cost tie {key}", _tie_image(*TIE_SEEDS[key]), {key: 1}) for key in TIE_SEEDS]


def seams(rng):
    """Stretches against the scans' 2 048-position tiles and the 16 383-symbol blocks, in a run-
    free stream: stretches whose first equal byte is at 2048k, 2048k - 1 and 2048k + 1, one
    ending at a seam, one across three tiles; stretch lengths 258m + 0, 1, 2, 3; the 16 383rd
    symbol a 258-match on a tile's first and on a tile's last position; a match as a block's
    first and as its last symbol."""
    out = []
    n = 9 * TILE + 2
    s = noise(rng, n, 0)
    s[0] = 1

    def run(a, length):                 # positions a .. a + length - 1 equal to s[a - 1]
        s[a:a + length] = s[a - 1]
        if a + length < n and s[a + length] == s[a - 1]:
            s[a + length] = s[a - 1] ^ 0x55

    run(TILE, 258)                      # starts on a tile, 258 * 1 + 0
    run(2 * TILE - 1, 259)              # one before a tile, 258 + 1
    run(3 * TILE + 1, 260)              # one after a tile, 258 + 2
    run(4 * TILE - 300, 300)            # ends on a seam
    run(5 * TILE - 5, 2 * TILE + 10)    # three tiles (and 258 * 16 + 78)
    run(8 * TILE + 100, 2 * 258 + 3)    # 258 * 2 + 3
    out.append(Case("tile seams", row_image(s[:n - (n - 1) % 3]),
                    {"stretch_at_tile": 1, "stretch_at_tile_m1": 1, "stretch_at_tile_p1": 1,
                     "stretch_ends_at_tile": 1, "stretch_3_tiles": 1, "stretch_258m_r0": 1,
                     "stretch_258m_r1": 1, "stretch_258m_r2": 1, "stretch_258m_r3": 1}))
    # the 16383rd symbol a 258-match starting on a tile's first / last position: literals up to
    # the match (symbol index 16382 at position p), so p - 16382 positions must be inside
    # earlier matches; one earlier stretch of that many bytes (whole 258s) does it
    for p, key in [(9 * TILE, "sym16383_match_tile_first"), (9 * TILE - 1,
                                                            "sym16383_match_tile_last")]:
        extra = p - (SYMS - 1)           # positions inside matches before p
        m, r = divmod(extra, 257)        # a stretch of 258j + r' bytes: j matches, j*257 inner
        s = noise(rng, p + 2 * 258 + 600, 0)
        s[0] = 1
        # stretch lengths of 258 give 257 inner positions each; the rest as a stretch of r + 1
        a = 1000
        for _ in range(m):
            s[a:a + 258] = s[a - 1]
            s[a + 258] = s[a - 1] ^ 0x33
            a += 300
        if r:
            s[a:a + r + 1] = s[a - 1]            # r + 1 bytes: one match of r + 1, r inner
            s[a + r + 1] = s[a - 1] ^ 0x33
        s[p:p + 258] = s[p - 1]                  # the block's last symbol: a 258-match at p
        s[p + 258:p + 2 * 258 + 1] = s[p - 1]    # and the next block's first: another stretch
        s[p + 2 * 258 + 1] = s[p - 1] ^ 0x77
        k = len(s) - (len(s) - 1) % 3
        out.append(Case(key, row_image(s[:k]), {key: 1, "match_first_in_block": 1,
                                                "match_last_in_block": 1}))
    return out


def _coded_counts(rng):
    """Literal counts of one full block on 16 values, skewed at random."""
    w = rng.random(16) ** 3 + 0.05
    c = np.floor(w / w.sum() * SYMS).astype(int)
    c[0] += SYMS - c.sum()
    return {1 + 7 * i: int(x) for i, x in enumerate(c)}


def stored_phases(rng):
    """Stored blocks after a coded block that ends at each of the 8 bit phases, then two stored
    blocks in a row, the second the final block.  Every coded block starts byte-aligned (after a
    stored block, or first), so its bit count mod 8 is the phase; the counts are drawn until each
    phase is met."""
    by_phase = {}
    while len(by_phase) < 8:
        c = _coded_counts(rng)
        lf = [0] * P.L_CODES
        for v, x in c.items():
            lf[v] = x
        lf[P.END_BLOCK] = 1
        b = P.block_trees(lf, [0] * P.D_CODES, SYMS, True)
        if b.type == P.STORED:
            continue
        bits = 3 + (b.hdr_bits if b.type == P.DYNAMIC else 0) + \
            sum(x * l for x, l in zip(lf, b.llen))
        by_phase.setdefault(bits % 8, c)
    parts, prev = [], 0
    for ph in range(8):
        c = by_phase[ph]
        a = ordered(c, prev) if parts else with_filter_byte(c)
        z = noise(rng, SYMS, a[-1])
        parts += [a, z]
        prev = z[-1]
    parts += [noise(rng, SYMS, prev)]
    parts += [noise(rng, 5000, parts[-1][-1])]
    return [Case("stored after 8 bit phases", row_image(pad_row(rng, parts)),
                 {**{f"stored_phase_{k}": 1 for k in range(8)}, "stored_stored": 1,
                  "stored_final": 1})]


def _zlen_stored(n):
    """zlen of a run-free stream of n bytes coded as stored blocks only (n % 16383 != 0)."""
    return 2 + n + 5 * (n // SYMS + 1) + 4


# (seed, W) of a one-row image of 64 levels whose zlib stream is exactly 8192 bytes; see chunks
ONE_CHUNK = (0, 3603)


def chunks(rng):
    """Zlib streams of length 0, 1, 2, 3, 4 and 8191 mod 8192, from run-free noise sized so
    that every block is stored (so zlen = n + 6 + 5 * blocks); with 1, 2 or 3 the Adler-32
    trailer straddles two IDAT chunks.  And one file of exactly one full chunk: a stored block
    of 8 181 bytes would do, but 8181 = 3^4 * 101 has no factor 3W + 1 > 1, so it is a coded
    one-row image found by a seeded search."""
    out = []
    for r in (0, 1, 2, 3, 4, 8191):
        for h in range(1, 60):
            hit = [W for W in range(2, 9000) if (h * (3 * W + 1)) % SYMS and
                   _zlen_stored(h * (3 * W + 1)) % 8192 == r and h * (3 * W + 1) > 8192]
            if hit:
                W = hit[0]
                break
        f = np.concatenate([np.concatenate([[1], noise(rng, 3 * W, 1)]) for _ in range(h)])
        for i in range(1, len(f)):
            assert f[i] != f[i - 1] or i % (3 * W + 1) == 0
        img = png_inputs.image_from_stream(f.reshape(h, 3 * W + 1)[:, 1:], h, W)
        out.append(Case(f"zlen {r} mod 8192", img, {f"zlen_mod_{r}": 1}))
    if ONE_CHUNK:
        seed, W = ONE_CHUNK
        out.append(Case("one chunk", _levels_row(seed, W), {"one_chunk": 1}))
    return out


def _levels_row(seed, W):
    r = np.random.default_rng(seed)
    return (r.integers(0, 64, (1, W, 3)) * 4).astype(np.uint8)


def adler(rng):
    """Streams of n = 65 521 (h = 1, W = 21 840), 65 520 (4 095 rows of W = 5) and 65 522 (two rows
    of W = 10 920) bytes, so n mod 65 521 is 0, -1 and 1 in the checksum's n - i weights; all of
    them 255 but the filter bytes, 32 and more tiles of the largest byte.  And n = 65 521 of
    noise."""
    out = []
    for n, h, W, key in [(65521, 1, 21840, "adler_n_0"), (65520, 4095, 5, "adler_n_m1"),
                         (65522, 2, 10920, "adler_n_p1")]:
        assert h * (3 * W + 1) == n
        img = png_inputs.image_from_stream(np.full((h, 3 * W), 255, np.uint8), h, W)
        out.append(Case(f"all 255, n = {n}", img, {key: 1, "adler_255_tiles": 32}))
    s = noise(rng, 65521, 0)
    s[0] = 1
    out.append(Case("noise, n = 65521", row_image(s), {"adler_n_0": 1}))
    return out


BUILDERS = [literal_overflow, bitlength_overflow, dummies, cost_ties, seams, stored_phases,
            chunks, adler]


def all_cases(seed=0):
    return [c for b in BUILDERS for c in b(np.random.default_rng(seed))]


# ------------------------------------------------------------------ census
def census(e):
    """Counts of every edge above in the oracle's encoding `e` (png_oracle.encode(img)[1])."""
    n = Counter()
    s = e.stream.astype(np.int64)
    nb = len(e.blocks)
    for k, b in enumerate(e.blocks):
        stats = {}
        P.block_trees(b.lfreq, b.dfreq, b.stored_len, b.can_store, stats=stats)
        ovf = stats["lit"]["overflow"]
        if ovf:
            n[f"lit_overflow_{ovf}"] += 1
            n["lit_overflow_first" if k == 0 and nb > 1 else
              "lit_overflow_final" if k == nb - 1 else "lit_overflow_middle"] += 1
            n["lit_overflow_full"] += b.nsym == SYMS
        if stats["bl"]["overflow"]:
            n[f"bl_overflow_{stats['bl']['overflow']}"] += 1
        for t in ("lit", "dist", "bl"):
            n["depth_tie"] += stats[t]["depth_tie"]
            n["full_tie"] += stats[t]["full_tie"]
        n["bl_single"] += sum(x > 0 for x in b.blfreq) == 1
        if b.type != P.STORED:
            n["dist_empty"] += b.dfreq[0] == 0 and b.nsym > 0
            n["dist_one"] += b.dfreq[0] > 0
        n["eob_only"] += b.nsym == 0
        n["one_literal_eob"] += sum(x > 0 for x in b.lfreq) == 2 and b.lfreq[P.END_BLOCK] == 1 \
            and all(x == 0 for x in b.lfreq[257:])
        d = b.stored_len + 4 - b.opt_lenb
        if b.can_store:
            n["stored_tie"] += d == 0
            n["stored_tie_m1"] += d == -1
            n["stored_tie_p1"] += d == 1
        if b.type != P.STORED:
            n[{0: "static_tie", -1: "static_tie_m1", 1: "static_tie_p1"}.get(
                b.static_lenb - b.dyn_lenb, "")] += 1
        n["hdr_bits_max"] = max(n["hdr_bits_max"], b.hdr_bits)
        if b.type == P.STORED and k > 0 and e.blocks[k - 1].type != P.STORED:
            n[f"stored_phase_{b.bit_start % 8}"] += 1
        n["stored_stored"] += b.type == P.STORED and k > 0 and e.blocks[k - 1].type == P.STORED
        n["stored_final"] += b.type == P.STORED and k == nb - 1
        if b.nsym:
            first = b.start
            last = max(i for i in range(max(b.start, b.end - MAX), b.end) if e.sym[i] >= 0)
            n["match_first_in_block"] += e.sym[first] >= 256
            n["match_last_in_block"] += e.sym[last] >= 256
            if b.nsym == SYMS and e.sym[last] == 256 + 255:
                n["sym16383_match_tile_first"] += last % TILE == 0
                n["sym16383_match_tile_last"] += last % TILE == TILE - 1
    n.pop("", None)
    # stretches: maximal runs of bytes equal to their predecessor, [a, z)
    eq = np.zeros(len(s), bool)
    eq[1:] = s[1:] == s[:-1]
    d = np.diff(np.concatenate([[0], eq.view(np.int8), [0]]))
    for a, z in zip(np.flatnonzero(d == 1), np.flatnonzero(d == -1)):
        n["stretch_at_tile"] += a % TILE == 0
        n["stretch_at_tile_m1"] += a % TILE == TILE - 1
        n["stretch_at_tile_p1"] += a % TILE == 1
        n["stretch_ends_at_tile"] += z % TILE == 0
        n["stretch_3_tiles"] += (z - 1) // TILE - a // TILE >= 2
        if z - a >= 258:
            n[f"stretch_258m_r{(z - a) % 258}"] += (z - a) % 258 <= 3
    zlen = len(e.zstream)
    n[f"zlen_mod_{zlen % 8192}"] += 1
    n["one_chunk"] += zlen == 8192
    ln = len(s)
    n[{0: "adler_n_0", MOD - 1: "adler_n_m1", 1: "adler_n_p1"}.get(ln % MOD, "")] += ln >= MOD - 1
    n.pop("", None)
    body = s[np.arange(ln) % (e.rowlen) != 0] if e.rowlen > 1 else s
    if len(body) and (body == 255).all():
        n["adler_255_tiles"] += -(-ln // TILE)
    return n

