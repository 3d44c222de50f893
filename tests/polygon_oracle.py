"""CPU restatement of pycocotools' polygon rasterisation: `annToRLE` of a polygon or box-list
annotation (`frPyObjects` on a list, `rleFrBbox`, `rleFrPoly`, `rleMerge`), returning the run
lists pycocotools would.  TEST INFRASTRUCTURE ONLY.

*** PARITY UNPINNED ***  pycocotools is not installed here.  These functions restate the
published C (pycocotools maskApi.c rleFrPoly / rleFrBbox / rleMerge, _mask.pyx frPyObjects,
coco.py annToRLE) loop for loop with C semantics: `int()` truncates toward zero as a C cast does,
every double operation is a separate Python float operation (no fused multiply-add), and a
zero-length edge takes s = 0 where C divides 0 by 0 (its one point never decides a toggle).
Positions are exact Python ints, where C's int positions overflow once H*W >= 2^31.
"""
import math
from fractions import Fraction

import numpy as np


def scale(c, floor=False):
    """[rleFrPoly] a vertex coordinate as (int)(5.0 * c + .5): two roundings, then truncation
    toward zero (`floor`, a model of a mistake, floors)."""
    z = 5.0 * float(c) + .5
    return math.floor(z) if floor else int(z)


def _minor(a, s, t, fused):
    """(int)(a + s*t + .5) with one rounding per operation; `fused`: a + s*t rounded once (FMA)."""
    if fused:
        return int(float(Fraction(a) + Fraction(s) * t) + .5)
    return int(a + s * t + .5)


class Edge:
    """One edge of rleFrPoly's walk from scaled vertex (xa, ya) to (xb, yb): the endpoints swapped
    when walking backwards, points t = 0 .. n emitted in the original direction.  `recip` models
    s = diff * (1/n) in place of diff / n; `fused` the minor coordinate as an FMA."""

    def __init__(self, xa, ya, xb, yb, recip=False, fused=False):
        dx, dy = abs(xb - xa), abs(ya - yb)
        self.xmaj = dx >= dy
        self.flip = (self.xmaj and xa > xb) or (not self.xmaj and ya > yb)
        xs, xe, ys, ye = (xb, xa, yb, ya) if self.flip else (xa, xb, ya, yb)
        self.xs, self.xe, self.ys, self.ye = xs, xe, ys, ye
        self.n = dx if self.xmaj else dy
        diff = ye - ys if self.xmaj else xe - xs
        if self.n == 0:
            self.s = 0.0
        elif recip:
            self.s = float(diff) * (1.0 / self.n)
        else:
            self.s = float(diff) / self.n
        self.fused = fused

    def u(self, t):
        return t + self.xs if self.xmaj else _minor(self.xs, self.s, t, self.fused)

    def v(self, t):
        return _minor(self.ys, self.s, t, self.fused) if self.xmaj else t + self.ys

    def window(self, lo, hi):
        """The t (ascending) of the points to walk when only u in [lo, hi] matters: for an
        x-major edge every t with u in [lo, hi]; for a y-major one, u being monotone in t, the
        first and the last t of each run of equal u in [lo, hi] (found by bisection on u(t)), so
        every pair where u changes is kept and a pair of kept points that were not neighbours
        has equal u."""
        n = self.n
        if self.xmaj:
            return range(max(0, lo - self.xs), min(n, hi - self.xs) + 1)
        sign = 1 if self.s >= 0.0 else -1

        def first(k):               # the first t in [0, n + 1) with sign * u(t) >= k
            a, b = 0, n + 1
            while a < b:
                m = (a + b) // 2
                if sign * self.u(m) >= k:
                    b = m
                else:
                    a = m + 1
            return a
        ends = (lo, hi) if sign > 0 else (-hi, -lo)
        ta, tb = first(ends[0]), first(ends[1] + 1) - 1
        if ta > tb:
            return []
        ts = {ta, tb}
        for k in range(sign * self.u(ta) + 1, sign * self.u(tb) + 1):
            t = first(k)
            ts |= {t - 1, t}
        return sorted(ts)


def scaled_vertices(xy, floor=False):
    """The scaled, closed vertex lists (x, y) of a part (an odd trailing number dropped)."""
    k = len(xy) // 2
    x = [scale(xy[2 * j], floor) for j in range(k)]
    y = [scale(xy[2 * j + 1], floor) for j in range(k)]
    return x + x[:1], y + y[:1]


def walk(x, y, recip=False, fused=False, window=None):
    """[rleFrPoly] the dense walk of the closed scaled polygon: lists u, v, the edge of each
    point and whether that edge is x-major.  `window` = (lo, hi) keeps only the points
    `Edge.window` names: with lo <= 0 and hi >= 5W every in-image toggle is kept (its two points
    are neighbours with u in [1, 5W - 1]), and a pair the gaps create has equal u or xd < 2 or
    > 5W - 3, so `toggles` drops it; the walk then costs what the image is wide, not what the
    edges are long."""
    u, v, ej, xm = [], [], [], []
    for j in range(len(x) - 1):
        e = Edge(x[j], y[j], x[j + 1], y[j + 1], recip, fused)
        ts = range(e.n + 1) if window is None else e.window(*window)
        ts = ts[::-1] if e.flip else ts
        for t in ts:
            u.append(e.u(t))
            v.append(e.v(t))
        ej += [j] * len(ts)
        xm += [e.xmaj] * len(ts)
    return u, v, ej, xm


def toggles(u, v, ej, xm, h, w, row_up=False, clamp_h1=False, xmaj_first=False,
            row_late=False):
    """[rleFrPoly] the kept column changes of a walk, downsampled: a list of (xd, yd, k, vmin)
    with k the index of the pair's second point.  Variants model kernel mistakes: `row_up` the
    row as (vmin + 3) / 5, `clamp_h1` rows clamped at h - 1, `xmaj_first` an x-major pair's row
    from the point of the smaller u only, `row_late` every row one later (at most h)."""
    out = []
    for j in range(1, len(u)):
        if u[j] != u[j - 1]:
            xd = float(u[j] if u[j] < u[j - 1] else u[j] - 1)
            xd = (xd + .5) / 5.0 - .5
            if math.floor(xd) != xd or xd < 0 or xd > w - 1:
                continue
            vmin = v[j] if v[j] < v[j - 1] else v[j - 1]
            yd = (float(vmin) + .5) / 5.0 - .5
            if yd < 0:
                yd = 0
            elif yd > h:
                yd = h
            yd = math.ceil(yd)
            if xmaj_first and xm[j] and ej[j] == ej[j - 1]:
                vmin = v[j] if u[j] < u[j - 1] else v[j - 1]
            if row_up or clamp_h1 or xmaj_first or row_late:
                yd = 0 if vmin <= 2 else min(h - 1 if clamp_h1 else h,
                                             (vmin + (3 if row_up else 2)) // 5)
                if row_late:
                    yd = min(yd + 1, h)
            out.append((int(xd), int(yd), j, vmin))
    return out


def runs(tg, h, w):
    """[rleFrPoly] the toggles (xd, yd, ...) sorted into run lengths, zero-length runs merged."""
    a = sorted([xx * h + yy for xx, yy, *_ in tg] + [h * w])
    p = 0
    for j in range(len(a)):
        t = a[j]
        a[j] -= p
        p = t
    b = [a[0]]
    j = 1
    while j < len(a):
        if a[j] > 0:
            b.append(a[j])
            j += 1
        else:
            j += 1
            if j < len(a):
                b[-1] += a[j]
                j += 1
    return b


WALK_KEYS = ("recip", "fused", "window")
TOGGLE_KEYS = ("row_up", "clamp_h1", "xmaj_first", "row_late")
SCALE_KEYS = ("floor",)


def part_toggles(xy, h, w, **variant):
    """The in-image toggles of one polygon part xy = [x0, y0, ...] (see `toggles`);
    `window=True` walks only u in [-3, 5w + 3] (see `walk`)."""
    if variant.get("window") is True:
        variant["window"] = (-3, 5 * w + 3)
    x, y = scaled_vertices(xy, **{k: variant[k] for k in SCALE_KEYS if k in variant})
    return toggles(*walk(x, y, **{k: variant[k] for k in WALK_KEYS if k in variant}), h, w,
                   **{k: variant[k] for k in TOGGLE_KEYS if k in variant})


def fr_poly(xy, h, w, **variant):
    """[pycocotools maskApi.c rleFrPoly] run lengths (column-major, starting with zeros) of the
    polygon xy = [x0, y0, x1, y1, ...] (an odd trailing number is dropped) on an h x w image.
    The keyword variants (see `scale`, `walk`, `toggles`) model one mistake each; none given is
    pycocotools."""
    return runs(part_toggles(xy, h, w, **variant), h, w)


def fr_bbox(bb, h, w, box_first=False, **variant):
    """[pycocotools maskApi.c rleFrBbox] the box [x, y, bw, bh] as the polygon (x, y) (x, y+bh)
    (x+bw, y+bh) (x+bw, y).  `box_first` models the far corner scaled as scale(x) + scale(bw)
    instead of scale(x + bw)."""
    xs, ys = float(bb[0]), float(bb[1])
    xe, ye = xs + float(bb[2]), ys + float(bb[3])
    if variant.get("window") is True:
        variant["window"] = (-3, 5 * w + 3)
    if box_first:
        f = {k: variant.pop(k) for k in SCALE_KEYS if k in variant}
        x0, y0 = scale(xs, **f), scale(ys, **f)
        x1, y1 = x0 + scale(bb[2], **f), y0 + scale(bb[3], **f)
        return runs(toggles(*walk([x0, x0, x1, x1, x0], [y0, y1, y1, y0, y0],
                                  **{k: variant[k] for k in WALK_KEYS if k in variant}), h, w,
                            **{k: variant[k] for k in TOGGLE_KEYS if k in variant}), h, w)
    return fr_poly([xs, ys, xs, ye, xe, ye, xe, ys], h, w, **variant)


def merge(rles, h, w):
    """[pycocotools maskApi.c rleMerge, intersect = 0] the union of run lists of one h x w image,
    the C loop as it is: both lists are walked run against run and a count is emitted where the
    OR changes or both lists end."""
    if len(rles) == 1:
        return list(rles[0])
    cnts = list(rles[0])
    for B in rles[1:]:
        A = cnts
        ca, cb = A[0], B[0]
        v = va = vb = False
        cnts = []
        a = b = 1
        cc, ct = 0, 1
        while ct > 0:
            c = min(ca, cb)
            cc += c
            ct = 0
            ca -= c
            if not ca and a < len(A):
                ca = A[a]
                a += 1
                va = not va
            ct += ca
            cb -= c
            if not cb and b < len(B):
                cb = B[b]
                b += 1
                vb = not vb
            ct += cb
            vp = v
            v = va or vb
            if v != vp or ct == 0:
                cnts.append(cc)
                cc = 0
    return cnts


def fr_py_objects(segm, h, w, **variant):
    """[pycocotools _mask.pyx frPyObjects, list input] per part: boxes when the first part has 4
    numbers, polygons when it has more; anything else raises as pycocotools does."""
    if not isinstance(segm, list) or len(segm) == 0:
        raise ValueError("input type is not supported.")
    n0 = len(segm[0])
    if n0 == 4:
        if any(len(bb) != 4 for bb in segm):
            raise ValueError("boxes must have 4 numbers")   # NumPy's ragged-array error there
        return [fr_bbox(bb, h, w, **variant) for bb in segm]
    if n0 > 4:
        variant.pop("box_first", None)
        return [fr_poly(p, h, w, **variant) for p in segm]
    raise ValueError("input type is not supported.")


def ann_to_rle(segm, h, w, xor=False, **variant):
    """[pycocotools coco.py annToRLE] the run lengths of a polygon / box list annotation.  The
    keyword variants are `fr_poly`'s and `fr_bbox`'s; `xor` models the parts XORed, not ORed."""
    parts = fr_py_objects(segm, h, w, **variant)
    if xor:
        m = np.zeros((h, w), bool)
        for r in parts:
            m ^= decode(r, h, w)
        return encode(m)
    return merge(parts, h, w)


def encode(m):
    """Column-major run lengths, starting with zeros, of a bool [h, w] mask."""
    flat = m.T.ravel()
    bounds = np.concatenate([[0], np.flatnonzero(flat[1:] != flat[:-1]) + 1, [flat.size]])
    r = [int(c) for c in np.diff(bounds)]
    return [0] + r if flat.size and flat[0] else r


def decode(counts, h, w):
    """[pycocotools rleDecode] bool [h, w] of column-major run lengths starting with zeros."""
    flat = np.zeros(h * w, bool)
    p, val = 0, False
    for c in counts:
        flat[p:p + c] = val
        p += c
        val = not val
    return flat.reshape(w, h).T


def ann_to_mask(segm, h, w, **variant):
    return decode(ann_to_rle(segm, h, w, **variant), h, w)
