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

import numpy as np


def fr_poly(xy, h, w):
    """[pycocotools maskApi.c rleFrPoly] run lengths (column-major, starting with zeros) of the
    polygon xy = [x0, y0, x1, y1, ...] (an odd trailing number is dropped) on an h x w image."""
    k = len(xy) // 2
    scale = 5.0
    x = [int(scale * float(xy[2 * j]) + .5) for j in range(k)]
    y = [int(scale * float(xy[2 * j + 1]) + .5) for j in range(k)]
    x.append(x[0])
    y.append(y[0])
    u, v = [], []
    for j in range(k):
        xs, xe, ys, ye = x[j], x[j + 1], y[j], y[j + 1]
        dx, dy = abs(xe - xs), abs(ys - ye)
        flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
        if flip:
            xs, xe, ys, ye = xe, xs, ye, ys
        if dx >= dy:
            s = 0.0 if dx == 0 else float(ye - ys) / dx
            for d in range(dx + 1):
                t = dx - d if flip else d
                u.append(t + xs)
                v.append(int(ys + s * t + .5))
        else:
            s = float(xe - xs) / dy
            for d in range(dy + 1):
                t = dy - d if flip else d
                v.append(t + ys)
                u.append(int(xs + s * t + .5))
    # points where the walk changes column, downsampled
    px, py = [], []
    for j in range(1, len(u)):
        if u[j] != u[j - 1]:
            xd = float(u[j] if u[j] < u[j - 1] else u[j] - 1)
            xd = (xd + .5) / scale - .5
            if math.floor(xd) != xd or xd < 0 or xd > w - 1:
                continue
            yd = float(v[j] if v[j] < v[j - 1] else v[j - 1])
            yd = (yd + .5) / scale - .5
            if yd < 0:
                yd = 0
            elif yd > h:
                yd = h
            yd = math.ceil(yd)
            px.append(int(xd))
            py.append(int(yd))
    a = sorted([xx * h + yy for xx, yy in zip(px, py)] + [h * w])
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


def fr_bbox(bb, h, w):
    """[pycocotools maskApi.c rleFrBbox] the box [x, y, bw, bh] as the polygon (x, y) (x, y+bh)
    (x+bw, y+bh) (x+bw, y)."""
    xs, ys = float(bb[0]), float(bb[1])
    xe, ye = xs + float(bb[2]), ys + float(bb[3])
    return fr_poly([xs, ys, xs, ye, xe, ye, xe, ys], h, w)


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


def fr_py_objects(segm, h, w):
    """[pycocotools _mask.pyx frPyObjects, list input] per part: boxes when the first part has 4
    numbers, polygons when it has more; anything else raises as pycocotools does."""
    if not isinstance(segm, list) or len(segm) == 0:
        raise ValueError("input type is not supported.")
    n0 = len(segm[0])
    if n0 == 4:
        if any(len(bb) != 4 for bb in segm):
            raise ValueError("boxes must have 4 numbers")   # NumPy's ragged-array error there
        return [fr_bbox(bb, h, w) for bb in segm]
    if n0 > 4:
        return [fr_poly(p, h, w) for p in segm]
    raise ValueError("input type is not supported.")


def ann_to_rle(segm, h, w):
    """[pycocotools coco.py annToRLE] the run lengths of a polygon / box list annotation."""
    return merge(fr_py_objects(segm, h, w), h, w)


def decode(counts, h, w):
    """[pycocotools rleDecode] bool [h, w] of column-major run lengths starting with zeros."""
    flat = np.zeros(h * w, bool)
    p, val = 0, False
    for c in counts:
        flat[p:p + c] = val
        p += c
        val = not val
    return flat.reshape(w, h).T


def ann_to_mask(segm, h, w):
    return decode(ann_to_rle(segm, h, w), h, w)
