"""Masks and regions built to sit on the edges where the contour tracer (csrc/contours.cu, DESIGN
§3.11) can stop matching find_contours, for tests/test_contour_edge_oracle.py (CPU) and
tests/test_gpu_contour_edges.py.

A batch is {"name", "planes": [bool [R, H_b, W_b] per image], "regions": int32 [B, R, 4] (y1, x1,
y2, x2), "counts": [B]}: instance k of image b is traced when k < counts[b], inside its region
clamped to the image.  Each builder returns {"batches": [...], "expect": {census key: minimum
count}}; `census` recounts what the batches hold, so an edit that drops an edge fails on the CPU.

The edges, by the tracer's structure (a lane owns the 32 cells c with (c - x1) // 32 == w, its
window adds one cell each side; a warp walks 32 words, 1024 cells, per chunk):
  * saddles (cases 6 and 9) at window positions 0, 1, 32 and 33 and on a chunk seam, for every
    x1 mod 8 (the byte phase of the region's first pixel);
  * cut regions: outside the image on each side, empty, 1 x 1, the whole image;
  * cycle lengths 2^k - 2, 2^k and 2^k + 2 as the longest instance of a call (the pointer-jumping
    rounds are ceil(log2(max_inst_segments))), and an instance far longer than its cycles;
  * totals S around the 4096-segment scan tile and cycle heads on segments 4094 and 4096.
"""
from collections import Counter

import numpy as np

import contour_oracle as co

WORD, CHUNK, TILE = 32, 1024, 4096


# ----------------------------------------------------------------------------- shapes
def checkerboard(H, W, parity=1):
    """Pixel (y, x) set where (y + x) % 2 == parity: every cell inside is a saddle."""
    return (np.indices((H, W)).sum(0) % 2 == parity)


def noise(rng, H, W, p=0.5):
    return rng.random((H, W)) < p


def rectangle(h, w, pad=1):
    """A filled h x w rectangle with `pad` zero pixels around it: one cycle of 2(h + w)."""
    m = np.zeros((h + 2 * pad, w + 2 * pad), bool)
    m[pad:pad + h, pad:pad + w] = True
    return m


def snake(n, run, pad=1):
    """A one-pixel-wide boustrophedon path of n pixels, runs of `run` pixels on even rows joined
    by one pixel on odd rows: no 2 x 2 block, no diagonal contact, so one cycle of 2n + 2."""
    left = True
    x, y, cells = 0, 0, []
    while len(cells) < n:
        xs = range(run) if left else range(run - 1, -1, -1)
        for x in xs:
            if len(cells) == n:
                break
            cells.append((y, x))
        if len(cells) < n:
            cells.append((y + 1, x))
        y += 2
        left = not left
    ys, xs = np.array(cells).T
    m = np.zeros((ys.max() + 1 + 2 * pad, run + 2 * pad), bool)
    m[ys + pad, xs + pad] = True
    return m


def dots(n_seg, width):
    """Isolated pixels (4 segments each) on a grid of pitch 2, plus one horizontal domino (6)
    when n_seg % 4 == 2: exactly n_seg segments, every cycle in rows of its own pixels."""
    assert n_seg % 2 == 0 and n_seg >= 4 and n_seg != 2
    n_dots, domino = (n_seg // 4, False) if n_seg % 4 == 0 else ((n_seg - 6) // 4, True)
    per_row = width // 2
    rows = (n_dots + per_row - 1) // per_row + 1
    m = np.zeros((2 * rows + 1, 2 * per_row + 2), bool)
    i = np.arange(n_dots)
    m[1 + 2 * (i // per_row), 1 + 2 * (i % per_row)] = True
    if domino:
        m[2 * rows - 1, 1:3] = True
    return m


def place(plane_hw, shape, y, x):
    m = np.zeros(plane_hw, bool)
    m[y:y + shape.shape[0], x:x + shape.shape[1]] = shape
    return m


def batch(name, planes, regions, counts=None):
    R = max(p.shape[0] for p in planes)
    planes = [np.concatenate([p, np.zeros((R - p.shape[0],) + p.shape[1:], bool)]) for p in planes]
    regions = np.asarray(regions, np.int32).reshape(len(planes), R, 4)
    counts = [R] * len(planes) if counts is None else list(counts)
    return {"name": name, "planes": planes, "regions": regions, "counts": counts}


def full(planes):
    """Regions covering each whole image."""
    return [[(0, 0, p.shape[1], p.shape[2])] * p.shape[0] for p in planes]


# ----------------------------------------------------------------------------- reference
def clamp(region, H, W):
    """The region as the tracer clamps it; None when empty."""
    y1, x1, y2, x2 = (int(v) for v in region)
    y1, x1, y2, x2 = max(y1, 0), max(x1, 0), min(y2, H), min(x2, W)
    return None if y2 <= y1 or x2 <= x1 else (y1, x1, y2, x2)


def cut(mask, region):
    """The mask zeroed outside its clamped region (all zero for an empty one)."""
    out = np.zeros_like(mask, dtype=bool)
    g = clamp(region, *mask.shape)
    if g is not None:
        y1, x1, y2, x2 = g
        out[y1:y2, x1:x2] = mask[y1:y2, x1:x2]
    return out


def reference(mask, region):
    """contour_oracle.mask_polygons of the mask zeroed outside the clamped region."""
    m = cut(mask, region)
    return co.mask_polygons(np.ones((1, 4), np.int32), m[:, :, None])[0]


def instances(b):
    """(image, k, mask, region) of every traced instance of batch b, in instance order."""
    for i, (planes, regs) in enumerate(zip(b["planes"], b["regions"])):
        for k in range(b["counts"][i]):
            yield i, k, planes[k], regs[k]


# ----------------------------------------------------------------------------- closed forms
DIAMOND = np.array([(0, .5), (-.5, 0), (0, -.5), (.5, 0), (0, .5)])


def dots_polygons(mask):
    """The polygons of a mask whose set pixels are all isolated (no 4- or 8-neighbour set): one
    diamond per pixel, in raster order, as flat (vertices [5 n, 2], contour offsets [n + 1])."""
    ys, xs = np.nonzero(mask)
    verts = (np.stack([xs, ys], 1).astype(np.float64)[:, None, :] + DIAMOND[None]).reshape(-1, 2)
    return verts, 5 * np.arange(ys.size + 1, dtype=np.int64)


def checkerboard_polygons(H, W, parity=1):
    """`dots_polygons` of `checkerboard(H, W, parity)` without building the mask: saddles keep
    diagonal pixels apart (vertex_connect_high=False), so every pixel is a diamond."""
    y = np.repeat(np.arange(H, dtype=np.int64), (W + ((np.arange(H) + parity + 1) % 2)) // 2)
    x0 = (y + parity) % 2
    start = np.concatenate([[0], np.cumsum(np.bincount(y, minlength=H))[:-1]])
    x = x0 + 2 * (np.arange(y.size) - start[y])
    verts = np.empty((y.size, 5, 2))
    verts[:, :, 0] = x[:, None] + DIAMOND[:, 0]
    verts[:, :, 1] = y[:, None] + DIAMOND[:, 1]
    return verts.reshape(-1, 2), 5 * np.arange(y.size + 1, dtype=np.int64)


def far_apart_reference(mask, blobs):
    """The oracle's polygons of a mask whose set pixels lie in the windows `blobs` [(y0, x0, y1,
    x1)], listed in raster order and far enough apart that no cell row or column of one touches
    another's: the oracle on each window, shifted, concatenated."""
    out = []
    for y0, x0, y1, x1 in blobs:
        sub = mask[y0:y1, x0:x1]
        for v in co.mask_polygons(np.ones((1, 4), np.int32), sub[:, :, None])[0]:
            out.append(v + np.array([x0, y0], np.float64))
    return out


# ----------------------------------------------------------------------------- census
def cells(mask, region):
    """Cases [rows, cols] of the traced cells (y2 - y1 + 1) x (x2 - x1 + 1) of the clamped
    region, and its x1; (None, None) when nothing is traced."""
    g = clamp(region, *mask.shape)
    if g is None:
        return None, None
    y1, x1, y2, x2 = g
    p = np.zeros((y2 - y1 + 2, x2 - x1 + 2), np.uint8)
    p[1:-1, 1:-1] = mask[y1:y2, x1:x2]
    case = p[:-1, :-1] + 2 * p[:-1, 1:] + 4 * p[1:, :-1] + 8 * p[1:, 1:]
    return case, x1


def cycles(mask, region):
    """(segments, [(smallest local segment number, length)] per cycle) of one instance, numbered
    as the tracer numbers them."""
    case, _ = cells(mask, region)
    if case is None or not case.any():
        return 0, []
    segs = co._segments_fast(_window(mask, region), 0.5)
    key = lambda pt: np.rint(np.asarray(pt) * 2).astype(np.int64) @ np.array([1 << 32, 1])
    frm = key([s[0] for s in segs])
    to = key([s[1] for s in segs])
    order = np.argsort(frm)
    succ = order[np.searchsorted(frm[order], to)]
    assert np.array_equal(frm[succ], to)
    low, nxt = np.arange(len(segs)), succ
    for _ in range(int(np.ceil(np.log2(len(segs)))) + 1):
        low = np.minimum(low, low[nxt])
        nxt = nxt[nxt]
    heads, lengths = np.unique(low, return_counts=True)
    return len(segs), list(zip(heads.tolist(), lengths.tolist()))


def _window(mask, region):
    """The traced pixels with their zero ring, as find_contours sees them (float64)."""
    y1, x1, y2, x2 = clamp(region, *mask.shape)
    p = np.zeros((y2 - y1 + 2, x2 - x1 + 2))
    p[1:-1, 1:-1] = mask[y1:y2, x1:x2]
    return p


def near_pow2(L):
    """(k, d) with L == 2^k + d for d in (-2, 0, 2), or None."""
    for d in (-2, 0, 2):
        k = int(L - d).bit_length() - 1
        if L - d > 0 and (L - d) == 1 << k:
            return k, d
    return None


def census(batches):
    """Counter of the edges the batches hold (module docstring)."""
    c = Counter()
    for b in batches:
        H = [p.shape[1] for p in b["planes"]]
        W = [p.shape[2] for p in b["planes"]]
        R = b["regions"].shape[1]
        n_inst = len(b["planes"]) * R
        if n_inst > 256:
            c["batch: B*R > 256"] += 1
        if max(H) + 1 > min(H) + 1:
            c["batch: row pitch > H + 1"] += 1
        seg_counts, base, longest, heads = [], 0, 0, []
        for i, planes in enumerate(b["planes"]):
            for k in range(R):
                reg = b["regions"][i, k]
                traced = k < b["counts"][i]
                if traced:
                    _region_kinds(c, reg, H[i], W[i])
                S_k, cyc = cycles(planes[k], reg) if traced else (0, [])
                seg_counts.append(S_k)
                if traced:
                    _saddles(c, planes[k], reg)
                for h, L in cyc:
                    heads.append(base + h)
                    longest = max(longest, L)
                    assert L % 2 == 0, (b["name"], L)
                base += S_k
        S = base
        c[f"S even"] += S % 2 == 0
        if S == 0 and n_inst > 256:
            c["batch: S = 0, B*R > 256"] += 1
        if S and seg_counts[0] == 0:
            c["batch: no segments first"] += 1
        if S and seg_counts[-1] == 0:
            c["batch: no segments last"] += 1
        nz = np.flatnonzero(seg_counts)
        if nz.size and (np.asarray(seg_counts[nz[0]:nz[-1]]) == 0).any():
            c["batch: no segments in the middle"] += 1
        smax = max(seg_counts, default=0)
        if longest and smax == longest and near_pow2(longest):
            k, d = near_pow2(longest)
            c[f"rounds: longest cycle 2^{k}{d:+d} = max_inst_segments"] += 1
        if longest and smax >= 64 * longest:
            c["rounds: max_inst_segments >= 64 x longest cycle"] += 1
        if S in (TILE - 2, TILE, TILE + 2, 2 * TILE):
            c[f"S = {S}"] += 1
        if S > TILE + 2 and S % TILE in (2, TILE - 2):
            c[f"S = 4096 t {'+' if S % TILE == 2 else '-'} 2, t >= 2"] += 1
        for h in heads:
            if h in (TILE - 2, TILE):
                c[f"head on segment {h}"] += 1
    return c


def _region_kinds(c, reg, H, W):
    y1, x1, y2, x2 = (int(v) for v in reg)
    if y1 < 0:
        c["cut: y1 < 0"] += 1
    if x1 < 0:
        c["cut: x1 < 0"] += 1
    if y2 > H:
        c["cut: y2 > H"] += 1
    if x2 > W:
        c["cut: x2 > W"] += 1
    if y2 == y1:
        c["cut: y2 == y1"] += 1
    if y2 < y1:
        c["cut: y2 < y1"] += 1
    if y2 - y1 == 1 and x2 - x1 == 1 and 0 <= y1 < H and 0 <= x1 < W:
        c["cut: 1 x 1"] += 1
    if (y1, x1, y2, x2) == (0, 0, H, W):
        c["cut: whole image"] += 1
    if 0 < y1 and 0 < x1 and y2 < H and x2 < W and y1 < y2 and x1 < x2:
        c["cut: inside on every side"] += 1


def _saddles(c, mask, reg):
    case, x1 = cells(mask, reg)
    if case is None:
        return
    ncells = case.shape[1]
    _, cols = np.nonzero((case == 6) | (case == 9))
    kinds = case[(case == 6) | (case == 9)]
    off = cols                      # c - x1
    for q, o in zip(kinds.tolist(), off.tolist()):
        pos = o % WORD
        if pos == 0:
            c[f"saddle {q} at window 1, x1 % 8 = {x1 % 8}"] += 1
            if o > 0:
                c[f"saddle {q} at window 33, x1 % 8 = {x1 % 8}"] += 1
        if pos == WORD - 1:
            c[f"saddle {q} at window 32, x1 % 8 = {x1 % 8}"] += 1
            if o + 1 < ncells:
                c[f"saddle {q} at window 0, x1 % 8 = {x1 % 8}"] += 1
        if o % CHUNK in (0, CHUNK - 1) and o >= CHUNK - 1 and o + 1 < ncells:
            c[f"saddle {q} on a chunk seam"] += 1


# ----------------------------------------------------------------------------- builders
SEAM_WIDTHS = (31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 2049)


def seam_patterns(rows=5):
    """A. Checkerboards of both parities and density-0.5 noise under regions of every cell width in
    SEAM_WIDTHS, x1 = 3 + j for j in 0..7; the planes are set outside the region too."""
    rng = np.random.default_rng(1101)
    planes, regions = [], []
    for cw in SEAM_WIDTHS:
        W = 3 + 8 + cw + 4
        H = rows + 4
        ps, rs = [], []
        for j in range(8):
            x1 = 3 + j
            for pat in (checkerboard(H, W, 0), checkerboard(H, W, 1), noise(rng, H, W)):
                ps.append(pat)
                rs.append((2, x1, 2 + rows, x1 + cw - 1))     # cw cells: x2 - x1 + 1
        planes.append(np.stack(ps))
        regions.append(rs)
    expect = {}
    for q in (6, 9):
        for pos in (0, 1, 32, 33):
            for m in range(8):
                expect[f"saddle {q} at window {pos}, x1 % 8 = {m}"] = 8
        expect[f"saddle {q} on a chunk seam"] = 8
    return {"batches": [batch("seams", planes, regions)], "expect": expect}


def placed_saddles():
    """A. Lone diagonal pairs, so the saddle's segments are the only ones near it: case 6 (the
    pair / ) and case 9 (\\), each at (c - x1) % 32 in {31, 0} and % 1024 in {1023, 0}, for
    x1 = 8 + j, j in 0..7, over one region 2100 cells wide."""
    H, cw = 6, 2100
    planes, regions = [], []
    for j in range(8):
        x1 = 8 + j
        W = x1 + cw + 4
        ps = []
        for q in (6, 9):
            m = np.zeros((H, W), bool)
            for o in (31, 64, 95, 128, 1023, 1056, 2048, 2079):
                c, r = x1 + o, 3                                 # cell (r, c) = the saddle
                if q == 6:
                    m[r - 1, c] = m[r, c - 1] = True
                else:
                    m[r - 1, c - 1] = m[r, c] = True
            ps.append(m)
        planes.append(np.stack(ps))
        regions.append([(0, x1, H, x1 + cw - 1)] * 2)
    expect = {}
    for q in (6, 9):
        for pos in (0, 1, 32, 33):
            for m in range(8):
                expect[f"saddle {q} at window {pos}, x1 % 8 = {m}"] = 2
        expect[f"saddle {q} on a chunk seam"] = 16
    return {"batches": [batch("placed saddles", planes, regions)], "expect": expect}


def cut_regions():
    """B. Noise planes set everywhere, under regions cut on every side, empty, 1 x 1 and whole;
    24 images of different sizes (so row_pitch = max_h + 1 passes most images' H + 1) with R = 12
    (B*R = 288 > 256: contour_finish_kernel runs two blocks); counts below R, and instances with
    no segments first, in the middle and last.  A second batch traces nothing: S = 0, B*R = 300."""
    rng = np.random.default_rng(1102)
    R = 12
    planes, regions, counts = [], [], []
    for b in range(24):
        H, W = int(rng.integers(1, 40)), int(rng.integers(1, 70))
        if b == 0:
            H, W = 61, 77
        planes.append(noise(rng, R * H, W).reshape(R, H, W) | (rng.random((R, H, W)) < 0.2))
        regs = [
            (0, 0, 0, 0),                                    # empty first
            (-3, 2, H // 2 + 1, W - 1),
            (1, -5, H - 1, W // 2 + 1),
            (H // 3, 1, H + 7, W),
            (1, W // 3, H, W + 9),
            (2, 2, 2, W),                                    # y2 == y1: empty, in the middle
            (H - 1, 1, 1, W),                                # y2 < y1
            (H // 2, W // 2, H // 2 + 1, W // 2 + 1),        # 1 x 1
            (0, 0, H, W),
            (-4, -4, H + 4, W + 4),
            (1, 1, max(H - 1, 2), max(W - 1, 2)),
            (0, 0, 0, 0),                                    # empty last
        ]
        regions.append(regs)
        counts.append(R if b % 3 else int(rng.integers(R // 2, R)))
    big = batch("cut regions", planes, regions, counts)
    zero = batch("nothing traced", [np.zeros((100, 9, 13), bool)] * 3,
                 [[(0, 0, 9, 13)] * 100] * 3)
    expect = {k: 8 for k in ("cut: y1 < 0", "cut: x1 < 0", "cut: y2 > H", "cut: x2 > W",
                             "cut: y2 == y1", "cut: y2 < y1", "cut: 1 x 1", "cut: whole image",
                             "cut: inside on every side")}
    expect.update({"batch: B*R > 256": 2, "batch: row pitch > H + 1": 1,
                   "batch: S = 0, B*R > 256": 1, "batch: no segments first": 1,
                   "batch: no segments in the middle": 1, "batch: no segments last": 1})
    return {"batches": [big, zero], "expect": expect}


JUMP_KS = tuple(range(3, 18))


def jump_rounds(ks=JUMP_KS):
    """C. One call per length L in {2^k - 2, 2^k, 2^k + 2}: a rectangle and a snake of one cycle of
    L each, so L = max_inst_segments sets the rounds; and one instance of 4096 dots (S_i = 16384)
    beside a 4-segment one, so the rounds far outrun every cycle."""
    out = []
    expect = {}
    for k in ks:
        for d in (-2, 0, 2):
            L = (1 << k) + d
            if L < 4:
                continue
            half = L // 2                                     # h + w of the rectangle
            h = max(1, min(half - 1, [1, 3, 17][k % 3]))
            rect = rectangle(h, half - h)
            n = (L - 2) // 2                                  # snake pixels
            run = max(1, min(n, [16, 64, 255][(k + d) % 3]))
            sn = snake(n, run)
            planes = [rect[None], sn[None]]                  # two images, one instance each
            out.append(batch(f"L = {L}", planes, full(planes)))
            expect[f"rounds: longest cycle 2^{k}{d:+d} = max_inst_segments"] = 1
    many = dots(4 * 4096, 128)
    one = place(many.shape, rectangle(1, 1), 0, 0)
    out.append(batch("rounds past the cycles", [np.stack([many, one])], full([np.stack([many, one])])))
    expect["rounds: max_inst_segments >= 64 x longest cycle"] = 1
    return {"batches": out, "expect": expect}


def scan_tiles():
    """D. Totals S in {4094, 4096, 4098, 8192, 4096 t +- 2}; an instance of 4094 or 4096
    segments before another puts the next cycle head on segment 4094 or 4096."""
    sizes = [[TILE - 2], [TILE], [TILE - 2, 4], [TILE, TILE], [TILE - 2, 4, TILE],
             [TILE, TILE - 2], [TILE, TILE + 2], [TILE - 2, 2 * TILE], [TILE, 2 * TILE + 2],
             [TILE - 2, 4 * TILE + 4]]
    out = []
    for parts in sizes:
        shapes = [dots(n, 64 + 2 * i) for i, n in enumerate(parts)]
        H = max(s.shape[0] for s in shapes)
        W = max(s.shape[1] for s in shapes)
        planes = np.stack([place((H, W), s, 0, 0) for s in shapes])
        out.append(batch(f"S = {sum(parts)}", [planes], full([planes])))
    expect = {"S = 4094": 1, "S = 4096": 1, "S = 4098": 1, "S = 8192": 1,
              "S = 4096 t - 2, t >= 2": 2, "S = 4096 t + 2, t >= 2": 3,
              "head on segment 4094": 4, "head on segment 4096": 4}
    return {"batches": out, "expect": expect}


BUILDERS = {"seams": seam_patterns, "placed saddles": placed_saddles, "cut regions": cut_regions,
            "jump rounds": jump_rounds, "scan tiles": scan_tiles}


# ----------------------------------------------------------------------------- E: past 2^23
def long_masks():
    """E. One-pixel-thin masks longer than float32 holds halves (2^23) or integers (2^24)
    exactly, with a few pixels at both ends: [(name, mask, blobs)] for `far_apart_reference`."""
    out = []
    for n in ((1 << 23) + 40, (1 << 24) + 40):
        row = np.zeros((1, n), bool)
        row[0, [0, 1, 3, n - 5, n - 4, n - 1]] = True
        if n < 1 << 24:
            out.append((f"1 x {n}", row, [(0, 0, 1, 8), (0, n - 8, 1, n)]))
        out.append((f"{n} x 1", row.T.copy(), [(0, 0, 8, 1), (n - 8, 0, n, 1)]))
    return out
