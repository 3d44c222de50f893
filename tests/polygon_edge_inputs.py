"""Polygon annotations built to sit on the edges where the polygon rasteriser's bit-exact claim
(DESIGN §3.16) can break, for tests/test_polygon_edge_oracle.py (CPU) and
tests/test_gpu_polygon_edges.py.  Each builder returns {"images": [((H, W), [segm, ...]), ...],
"expect": {census key: minimum count}}; `census` counts what the inputs hold, so an edit that
drops an edge fails the CPU test instead of passing quietly.  Coordinates are given as the
doubles a JSON file would parse to; `at(k)` is the coordinate whose scaled value
(int)(5.0*c + .5) is exactly the integer k."""
import functools
import json
from collections import Counter

import polygon_oracle as po

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1


def at(k):
    """A coordinate that rleFrPoly scales back to exactly k: k / 5, or (k - 0.7) / 5 for k <= 0,
    where the truncation of 5c + .5 goes toward zero."""
    c = k / 5 if k > 0 else (k - 0.7) / 5
    assert po.scale(c) == k, k
    return c


def part(vs):
    """A polygon part [x0, y0, ...] from scaled integer vertices [(x, y), ...]."""
    return [at(c) for v in vs for c in v]


def shape_of(vs, pad=3):
    """An image that holds every toggle of the scaled vertices vs."""
    return (max(y for _, y in vs) // 5 + pad, max(x for x, _ in vs) // 5 + pad)


# ----------------------------------------------------------------------------- exact search
def _edge_triangle(xmaj, a, diff, n, flip, shift, far):
    """A triangle of scaled vertices whose first edge runs n along the major axis from minor
    coordinate a by diff (walked backwards when flip), closed by a vertex `far` away."""
    if xmaj:
        p, q, r = (shift, a), (shift + n, a + diff), (shift, a + far)
    else:
        p, q, r = (a, shift), (a + diff, shift + n), (a + far, shift)
    return [q, p, r] if flip else [p, q, r]


def _toggle_set(vs, H, W, **variant):
    x, y = [v[0] for v in vs] + [vs[0][0]], [v[1] for v in vs] + [vs[0][1]]
    return sorted(t[:2] for t in po.toggles(*po.walk(x, y, **variant), H, W))


@functools.lru_cache(maxsize=None)
def search_minor(variant, per_branch=3, n_max=60):
    """Exact search over small integer vertices for triangles whose toggles change under the
    walk variant `variant` ("fused": a + s*t rounded once, as an FMA would; "recip": s as
    diff * (1/n)).  Candidates are the (a, diff, n, t) where the variant's minor coordinate
    differs from (int)(a + s*t + .5) with one rounding per operation (for "fused", decided with
    Fraction arithmetic); each is put on an edge that is x-major or y-major, walked forwards or
    backwards, with a >= 0 or a < 0, and kept when the triangle's toggles differ.  Returns
    {(xmaj, flip, a < 0): [vertex lists]}, per_branch of each."""
    from fractions import Fraction
    found = {}
    for n in range(2, n_max):
        for diff in range(-n + 1, n):
            if diff == 0:
                continue
            s = diff / n
            s_var = diff * (1.0 / n) if variant == "recip" else s
            for t in range(1, n):
                if variant == "fused" and Fraction(s) * t == Fraction(s * t):
                    continue
                for a in range(-n - 3, n + 4):
                    if variant == "fused":
                        other = int(float(Fraction(a) + Fraction(s) * t) + .5)
                    else:
                        other = int(a + s_var * t + .5)
                    if int(a + s * t + .5) == other:
                        continue
                    for xmaj in (True, False):
                        for flip in (False, True):
                            got = found.setdefault((xmaj, flip, a < 0), [])
                            if len(got) >= per_branch:
                                continue
                            for shift in range(5, 10):
                                vs = next((vs for far in (40, -40)
                                           for vs in [_edge_triangle(xmaj, a, diff, n, flip,
                                                                     shift, far)]
                                           if vs not in got and
                                           _toggle_set(vs, *shape_of(vs)) !=
                                           _toggle_set(vs, *shape_of(vs), **{variant: True})),
                                          None)
                                if vs is not None:
                                    got.append(vs)
                                    break
        if len(found) == 8 and all(len(v) >= per_branch for v in found.values()):
            break
    return found


def unfused_minor():
    """Parts where (int)(a + s*t + .5) rounded once per operation and as an FMA give different
    masks: every branch (x-major and y-major walk, forwards and backwards, a >= 0 and a < 0),
    three each, each on its own image; and the 0.2-grid polygon of a random sweep where the two
    differ by one pixel."""
    images = [(shape_of(vs), [[part(vs)]])
              for _, parts in sorted(search_minor("fused").items()) for vs in parts]
    images.append(((12, 19), [[[15.8, -0.8, 7.6, 17.6, 2.8, 18.0, -0.8, 1.6]]]))
    return {"images": images, "expect": {"fused_parts": 25}}


def reciprocal_division():
    """Parts where s = diff / n and s = diff * (1/n) give different masks, every branch."""
    images = [(shape_of(vs), [[part(vs)]])
              for _, parts in sorted(search_minor("recip").items()) for vs in parts]
    return {"images": images, "expect": {"recip_parts": 24}}


# ----------------------------------------------------------------------------- scaling
TIES = ["0.3", "0.1", "0.7", "1.3", "2.5", "12.7", "-0.1", "-0.15", "-0.3", "-0.45", "7.9",
        "-0.7", "3.1"]


def scaling_ties():
    """Vertices at decimal coordinates as json.loads parses them whose 5.0*c rounds onto k + 0.5
    (0.3 -> 1.5 -> 2, where rounding half to even would give 2 from 2.5 and 1.5 alike), and
    negative ones where C truncation and floor differ (-0.15 -> 0, not -1), on edges that cross
    into the image."""
    c = [json.loads(s) for s in TIES]
    imgs = []
    for i, a in enumerate(c):
        b = c[(i + 3) % len(c)]
        imgs.append(((9, 11), [[[a, b, 6.3, b, 9.1, 7.7, a, 6.1]],
                               [[-0.15, a, 4.7, -0.1, 8.5, 4.3 + b, b, 5.9]],
                               [[a, -0.15, a + 5.1, -0.45, 3.7, 8.3]]]))
    return {"images": imgs, "expect": {"tie_vertices": 60, "trunc_not_floor": 40,
                                       "floor_instances": 8}}


# ----------------------------------------------------------------------------- rows
def toggle_rows():
    """Horizontal and sloped edges whose pair minimum vmin is = 2 and = 3 (mod 5), vmin <= 2 next
    to vmin = 3, rows clamped to H (H = 64 and H = 45) and rows 0, 31, 32 and H - 1, the band
    boundaries of poly_planes_kernel."""
    images = []
    for H in (64, 45):
        segs = []
        for r in (0, 1, 6, 30, 31, 32, 33, H - 2, H - 1):
            for dv in (0, 1, -4, -3):      # vmin = 5r + 2 + dv: = 2, 3, 3 (row r), 4
                top = 5 * r + 2 + dv
                segs.append([part([(7, top), (57, top), (57, top + 9), (7, top + 9)])])
        segs.append([part([(2, 2), (40, 3), (60, 2), (60, 5 * H + 30), (2, 5 * H + 9)])])
        segs.append([part([(12, -7), (37, 3), (52, 1), (52, 5 * H - 3), (12, 5 * H - 2)])])
        segs.append([part([(3, 5 * H - 8), (90, 5 * H - 7), (90, 5 * H + 3), (3, 5 * H + 2)])])
        images.append(((H, 21), segs))
    return {"images": images, "expect": {"vmin_2mod5": 20, "vmin_3mod5": 20, "vmin_le2": 4,
                                         "vmin_eq3": 4, "row_H": 10, "row_0": 4, "row_31": 4,
                                         "row_32": 4, "row_Hm1": 4, "row_up_instances": 10,
                                         "clamp_h1_instances": 2, "row_late_instances": 10}}


def both_minima():
    """x-major pairs (c, c + 1) whose two points round to rows on either side of a row boundary:
    v falling across the pair (the minimum is the point at c + 1) and v rising (at c), walked in
    both directions."""
    images = []
    for k in range(12):
        vs = [(2 + k, 20 + k), (75 + k, 55 - k), (40, 95 + 2 * k)]
        images.append((shape_of(vs), [[part(vs)], [part(vs[::-1])],
                                      [part([(5, 60), (70 + k, 29 + k), (88, 70)])]]))
    return {"images": images, "expect": {"xmaj_min_at_c": 30, "xmaj_min_at_c1": 15,
                                         "xmaj_first_instances": 10}}


def y_major():
    """y-major edges rising and falling in u, walked forwards and backwards (the same quad in
    both vertex orders), with the column change at t = 1 and at t = n - 1, and vertical edges
    (s = 0, u constant)."""
    images = []
    for k in range(6):
        c, n, y0 = 5 * (k + 1) + 2, 40 + 7 * k, 3 + k     # (c, c + 1) toggles column k + 1
        segs = []
        for a, b in [((c, y0), (c + n - 1, y0 + n)),          # rising, the change at t = 1
                     ((c + 2 - n, y0), (c + 1, y0 + n)),      # rising, at t = n - 1
                     ((c + 1, y0), (c + 2 - n, y0 + n)),      # falling, at t = 1
                     ((c + n - 1, y0), (c, y0 + n))]:         # falling, at t = n - 1
            vs = [a, b, (b[0] + 30, b[1]), (a[0] + 30, a[1])]
            segs += [[part(vs)], [part(vs[::-1])]]
        segs.append([part([(c, 1), (c, 80), (c + 25, 80), (c + 25, 1)])])
        images.append(((20, 14), segs))
    return {"images": images, "expect": {"ymaj_rise_fwd": 12, "ymaj_rise_back": 12,
                                         "ymaj_fall_fwd": 12, "ymaj_fall_back": 12,
                                         "ymaj_t1": 24, "ymaj_tn1": 24, "ymaj_s0_edges": 12}}


def cull_boundary():
    """Toggle pairs that end exactly on an edge's extreme vertex: c + 1 = max x and c = min x,
    on x-major and y-major edges, so a cull one unit tighter than the tightest correct one loses
    them."""
    images = []
    for X in range(1, 9):
        c = 5 * X + 2
        images.append(((16, 12), [[part([(c, 4), (c + 1, 40), (c - 20, 45)])],
                                  [part([(c + 1, 6), (c - 30, 20), (c - 10, 55)])],
                                  [part([(c, 9), (c + 40, 25), (c + 9, 60)])],
                                  [part([(c, 50), (c + 1, 12), (c + 30, 30)])]]))
    return {"images": images, "expect": {"cull_at_max": 16, "cull_at_min": 16}}


# ----------------------------------------------------------------------------- columns
def scan_seams():
    """Images W = 256, 257, 512, 513 and 3840 (passes of 256 columns in the toggles kernel's block
    scan) with toggles in columns 254-257 and 510-513 and parts that span the seams."""
    images = []
    for W in (256, 257, 512, 513, 3840):
        segs = []
        for X in (254, 255, 256, 257, 510, 511, 512, 513):
            if X < W:
                x = 5 * X
                segs.append([part([(x - 3, 10), (x + 4, 25), (x - 2, 40)]),
                             part([(x, 50), (x + 9, 57), (x, 99)])])
        segs.append([part([(3, 5), (5 * W - 3, 40), (5 * W - 40, 90), (7, 70)])])
        segs.append([part([(1100, 3), (1500, 80), (2700, 33), (2500, 7)])])
        images.append(((24, W), segs))
    return {"images": images, "expect": {"seam_256": 10, "seam_512": 6}}


def dense_toggles():
    """Sawtooth parts whose every edge has as many in-image toggles as an edge of its |dx| can
    have (min(W, (|dx| + 4) // 5)), and edges that span more than the image is wide."""
    images = []
    for W in (9, 40, 64):
        segs = []
        for step in (1, 2, 6, 7):       # |dx| = 1, 2 (mod 5): one more than (|dx| + 3) // 5
            x, top = 2, []
            while x + step <= 5 * W - 3:
                top += [(x, 3 + 17 * (len(top) % 2)), (x + step, 3 + 17 * (len(top) % 2))]
                x += 5 * ((step + 4) // 5)
            vs = top + [(x, 90), (2, 90)]
            segs.append([part(vs)])
        segs.append([part([(-500, 10), (5 * W + 500, 14), (5 * W + 600, 60), (-700, 70)])])
        segs.append([part([(-9000, 60), (5 * W + 7000, 61), (40, 99)])])
        images.append(((21, W), segs))
    return {"images": images, "expect": {"tight_edges": 60, "wide_edges": 6}}


def overlapping_parts():
    """Instances of two and three parts whose union differs from their XOR."""
    imgs = []
    for k in range(4):
        imgs.append(((30, 30), [[part([(0, 0), (60 + k, 0), (60, 70), (0, 60)]),
                                 part([(30, 30), (120, 33 + k), (100, 110), (35, 100)])],
                                [part([(5, 5), (100, 5), (100, 100)]),
                                 part([(5, 100), (100, 100), (5, 5)]),
                                 part([(50, 10), (140, 70), (10, 140)])]]))
    return {"images": imgs, "expect": {"xor_instances": 8}}


def box_lists():
    """[x, y, w, h] boxes where x + w in double scales to another integer than the scaled corner
    plus the scaled width would, and boxes on decimal ties."""
    vals = [json.loads(s) for s in ("0.1", "0.2", "0.3", "0.7", "1.1", "2.3", "4.9", "0.45")]
    imgs = []
    for i, a in enumerate(vals):
        b = vals[(i + 1) % len(vals)]
        imgs.append(((12, 12), [[[a, b, 3 * b + 1.3, 2 * a + 0.9]],
                                [[a + 1.1, 0.3, b + 4.7, a + 5.3], [b, a, 0.7, 1.3]],
                                [[-0.15, -0.3, b + 2.2, a + 3.4]]]))
    return {"images": imgs, "expect": {"box_first_instances": 6}}


# ----------------------------------------------------------------------------- int range
def int_range():
    """Scaled coordinates of exactly 2^31 - 1 and -2^31 and a consecutive difference of exactly
    2^31 - 1, all accepted, on edges that cross the image; `int_range_refused` gives one past
    each."""
    hi, lo = at(INT_MAX), at(INT_MIN)
    d0 = at(INT_MAX - (1 << 30))     # 2^30 - 1, so d0 - (-2^30) = 2^31 - 1
    m30 = at(-(1 << 30))
    segms = [[[hi, 3.3, 0.7, 9.1, 2.3, 0.4]],                     # dx = 2^31 - 1 - 3
             [[1.1, 0.2, hi, 7.7, 4.9, 10.3]],
             [[lo, 5.5, -0.4, 1.2, -0.4, 8.9]],
             [[m30, 0.9, d0, 8.2, 6.6, 10.1]],                  # the 2^31 - 1 difference
             [[2.1, m30, 5.7, d0, 8.8, 3.3]],
             [[0.5, hi, 3.2, 1.1, 7.4, 0.6]],
             [[9.9, lo, 9.3, -0.4, 0.2, -0.4]]]
    return {"images": [((13, 11), segms)], "expect": {"int_max": 3, "int_min": 2,
                                                    "diff_max": 2}}


def int_range_refused():
    """One past each accepted end: a scaled 2^31, a scaled -2^31 - 1, a difference of 2^31."""
    return [[[at(INT_MAX + 1), 1.0, 2.0, 3.0, 4.0, 5.0]],
            [[at(INT_MIN - 1), 1.0, 2.0, 3.0, 4.0, 5.0]],
            [[at(-1), 1.0, at(INT_MAX), 3.0, 4.0, 5.0]],
            [[0.0, at(INT_MIN), 1.0, at(0), 4.0, 5.0]]]


BIG_HW = (46341, 46341)     # H*W = 2^31 + 4633


def big_image():
    """One image with H*W >= 2^31, where pycocotools' int positions overflow: parts reaching its
    last columns and rows, so positions past 2^31 are toggled."""
    H, W = BIG_HW
    segms = [[[W - 30.3, H - 40.1, W + 5.0, H - 3.7, W - 3.3, H + 8.2, W - 60.7, H - 1.1]],
             [[10.0, 20.0, W - 12.6, 7.0, W - 1.4, H - 2.2, 3.0, H - 9.9],
              [W / 2, 1.0, W - 0.6, H / 3, W / 3, H / 2.5]]]
    return {"images": [((H, W), segms)], "expect": {}}


# ----------------------------------------------------------------------------- census
# the oracle variants (each a model of one mutant of tools/mutate_polygons.py) and the census key
# that counts the instances whose mask they change
VARIANTS = {"fused": {"fused": True}, "recip": {"recip": True}, "floor": {"floor": True},
            "row_up": {"row_up": True},
            "clamp_h1": {"clamp_h1": True}, "xmaj_first": {"xmaj_first": True},
            "row_late": {"row_late": True}, "xor": {"xor": True}, "box_first": {"box_first": True}}


def is_boxes(segm):
    return len(segm[0]) == 4


def edge_bound(dx, W):
    """The most in-image toggles one edge of |dx| scaled columns can hold: one per c = 5X + 2 in a
    range of dx consecutive pair starts, at most one per column."""
    return min(W, (dx + 4) // 5)


def census(images, variants=True):
    """Counts of the edges the builders target, over every toggle of every polygon part (the
    windowed walk; boxes count only for their instance variants)."""
    n = Counter()
    for (H, W), segms in images:
        for segm in segms:
            if variants:
                want = po.ann_to_mask(segm, H, W, window=True)
                for name, kw in VARIANTS.items():
                    if name == "box_first" and not is_boxes(segm):
                        continue
                    n[name + "_instances"] += not (want == po.ann_to_mask(segm, H, W, window=True,
                                                                          **kw)).all()
            if is_boxes(segm):
                continue
            for xy in segm:
                _part_census(n, xy, H, W, variants)
    return n


def _part_census(n, xy, H, W, variants):
    x, y = po.scaled_vertices(xy)
    k = len(x) - 1
    for j in range(len(xy) // 2 * 2):
        c = float(xy[j])
        n["tie_vertices"] += (5.0 * c) % 1 == .5
        n["trunc_not_floor"] += po.scale(c) != po.scale(c, floor=True)
    n["int_max"] += sum(c == INT_MAX for c in x[:k] + y[:k])
    n["int_min"] += sum(c == INT_MIN for c in x[:k] + y[:k])
    n["diff_max"] += sum(max(abs(x[j + 1] - x[j]), abs(y[j + 1] - y[j])) == INT_MAX
                         for j in range(k))
    edges = [po.Edge(x[j], y[j], x[j + 1], y[j + 1]) for j in range(k)]
    n["ymaj_s0_edges"] += sum(not e.xmaj and e.s == 0.0 and e.n > 0 for e in edges)
    u, v, ej, xm = po.walk(x, y, window=(-3, 5 * W + 3))
    tg = po.toggles(u, v, ej, xm, H, W)
    if variants:
        for name in ("fused", "recip"):
            n[name + "_parts"] += [t[:2] for t in tg] != [
                t[:2] for t in po.part_toggles(xy, H, W, window=True, **{name: True})]
    per_edge, per_col = Counter(), Counter()
    for xd, yd, i, vmin in tg:
        per_col[xd] += 1
        n["row_0"] += yd == 0
        n["row_31"] += yd == 31
        n["row_32"] += yd == 32
        n["row_Hm1"] += yd == H - 1
        n["row_H"] += yd == H
        n["vmin_le2"] += vmin <= 2
        n["vmin_eq3"] += vmin == 3
        n["vmin_2mod5"] += vmin > 2 and vmin % 5 == 2
        n["vmin_3mod5"] += vmin > 2 and vmin % 5 == 3
        n["seam_256"] += xd in (255, 256)
        n["seam_512"] += xd in (511, 512)
        if ej[i] != ej[i - 1]:
            n["junction"] += 1
            continue
        e = edges[ej[i]]
        per_edge[ej[i]] += 1
        c = 5 * xd + 2
        n["cull_at_max"] += c + 1 == max(e.xs, e.xe)
        n["cull_at_min"] += c == min(e.xs, e.xe)
        if e.xmaj:
            v_c, v_c1 = (v[i], v[i - 1]) if u[i] < u[i - 1] else (v[i - 1], v[i])
            row = [0 if q <= 2 else (q + 2) // 5 for q in (v_c, v_c1)]
            if row[0] != row[1]:
                n["xmaj_min_at_c" if v_c < v_c1 else "xmaj_min_at_c1"] += 1
        else:
            tmax = max(v[i], v[i - 1]) - e.ys
            n["ymaj_{}_{}".format("rise" if e.s >= 0.0 else "fall",
                                  "back" if e.flip else "fwd")] += 1
            n["ymaj_t1"] += tmax == 1
            n["ymaj_tn1"] += tmax == e.n
    for j, e in enumerate(edges):
        dx = abs(e.xe - e.xs)
        assert per_edge[j] <= edge_bound(dx, W), (xy, j)
        n["tight_edges"] += per_edge[j] > 0 and per_edge[j] == edge_bound(dx, W)
        n["wide_edges"] += dx > 5 * W and per_edge[j] == W
    n["odd_columns"] += sum(c % 2 for c in per_col.values())


BUILDERS = [unfused_minor, reciprocal_division, scaling_ties, toggle_rows, both_minima, y_major,
            cull_boundary, scan_seams, dense_toggles, overlapping_parts, box_lists, int_range]
