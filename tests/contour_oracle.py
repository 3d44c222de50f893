"""CPU restatement of the contour loop of `visualize.display_instances` (serve.py:160-169).
TEST INFRASTRUCTURE ONLY.

Upstream draws, for every instance whose box is not all zeros,

    padded_mask = np.zeros((H + 2, W + 2), dtype=np.uint8)
    padded_mask[1:-1, 1:-1] = masks[:, :, i]
    contours = skimage.measure.find_contours(padded_mask, 0.5)
    for verts in contours:
        verts = np.fliplr(verts) - 1

*** PARITY UNPINNED ***  scikit-image is not vendored by the reference and cannot be imported
here.  `find_contours` below restates skimage.measure.find_contours (fully_connected='low',
positive_orientation='low'): `_segments` is its marching-squares pass (`_get_contour_segments`,
vertex_connect_high=False) and `_assemble` its `_assemble_contours`.

`contours_by_cycles` is the closed form the device implements instead of the dictionary merges;
the tests check it against `_assemble`.
"""
from collections import deque

import numpy as np


def _fraction(a, b, level):
    if b == a:
        return 0.0
    return (level - a) / (b - a)


def _segments(image, level):
    """Marching squares: (from_point, to_point) pairs in raster order of the cells."""
    segs = []
    image = np.asarray(image, dtype=np.float64)
    for r0 in range(image.shape[0] - 1):
        for c0 in range(image.shape[1] - 1):
            r1, c1 = r0 + 1, c0 + 1
            ul, ur, ll, lr = image[r0, c0], image[r0, c1], image[r1, c0], image[r1, c1]
            case = (ul > level) + 2 * (ur > level) + 4 * (ll > level) + 8 * (lr > level)
            if case in (0, 15):
                continue
            top = (r0, c0 + _fraction(ul, ur, level))
            bottom = (r1, c0 + _fraction(ll, lr, level))
            left = (r0 + _fraction(ul, ll, level), c0)
            right = (r0 + _fraction(ur, lr, level), c1)
            if case == 1:
                segs.append((top, left))
            elif case == 2:
                segs.append((right, top))
            elif case == 3:
                segs.append((right, left))
            elif case == 4:
                segs.append((left, bottom))
            elif case == 5:
                segs.append((top, bottom))
            elif case == 6:                      # vertex_connect_high=False
                segs.append((right, top))
                segs.append((left, bottom))
            elif case == 7:
                segs.append((right, bottom))
            elif case == 8:
                segs.append((bottom, right))
            elif case == 9:                      # vertex_connect_high=False
                segs.append((top, left))
                segs.append((bottom, right))
            elif case == 10:
                segs.append((bottom, top))
            elif case == 11:
                segs.append((bottom, left))
            elif case == 12:
                segs.append((left, right))
            elif case == 13:
                segs.append((top, right))
            elif case == 14:
                segs.append((left, top))
    return segs


# (from edge, to edge) per case, edges 0 top 1 bottom 2 left 3 right; saddles' second segment
_FIRST = {1: (0, 2), 2: (3, 0), 3: (3, 2), 4: (2, 1), 5: (0, 1), 6: (3, 0), 7: (3, 1), 8: (1, 3),
          9: (0, 2), 10: (1, 0), 11: (1, 2), 12: (2, 3), 13: (0, 3), 14: (2, 0)}
_SECOND = {6: (2, 1), 9: (1, 3)}


def _segments_fast(image, level):
    """`_segments` with NumPy (same segments, same order)."""
    a = np.asarray(image, dtype=np.float64)
    ul, ur, ll, lr = a[:-1, :-1], a[:-1, 1:], a[1:, :-1], a[1:, 1:]
    case = (ul > level) + 2 * (ur > level) + 4 * (ll > level) + 8 * (lr > level)

    def frac(p, q):
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(q == p, 0.0, (level - p) / (q - p))

    r0, c0 = np.nonzero((case != 0) & (case != 15))
    q = case[r0, c0]
    r0f, c0f = r0.astype(np.float64), c0.astype(np.float64)
    pts = np.empty((4, r0.size, 2))
    pts[0] = np.stack([r0f, c0f + frac(ul, ur)[r0, c0]], 1)
    pts[1] = np.stack([r0f + 1, c0f + frac(ll, lr)[r0, c0]], 1)
    pts[2] = np.stack([r0f + frac(ul, ll)[r0, c0], c0f], 1)
    pts[3] = np.stack([r0f + frac(ur, lr)[r0, c0], c0f + 1], 1)
    fe = np.array([_FIRST.get(k, (0, 0))[0] for k in range(16)])[q]
    te = np.array([_FIRST.get(k, (0, 0))[1] for k in range(16)])[q]
    idx = np.arange(r0.size)
    first = list(zip(map(tuple, pts[fe, idx].tolist()), map(tuple, pts[te, idx].tolist())))
    sad = np.nonzero((q == 6) | (q == 9))[0]
    out, prev = [], 0
    for i in sad.tolist():
        out.extend(first[prev:i + 1])
        f2, t2 = _SECOND[int(q[i])]
        out.append((tuple(pts[f2, i].tolist()), tuple(pts[t2, i].tolist())))
        prev = i + 1
    out.extend(first[prev:])
    return out


def _assemble(segments):
    """Join segments into contours: the start / end dictionaries of `_assemble_contours`, merges
    keeping the contour created first, contours returned in creation order."""
    current = 0
    contours, starts, ends = {}, {}, {}
    for frm, to in segments:
        if frm == to:
            continue
        tail, tail_num = starts.pop(to, (None, None))
        head, head_num = ends.pop(frm, (None, None))
        if tail is not None and head is not None:
            if tail is head:
                head.append(to)                  # closes a contour
            elif tail_num > head_num:
                head.extend(tail)                # tail created second: append it to head
                contours.pop(tail_num, None)
                starts[head[0]] = (head, head_num)
                ends[head[-1]] = (head, head_num)
            else:
                tail.extendleft(reversed(head))  # head created second: prepend it to tail
                starts.pop(head[0], None)
                contours.pop(head_num, None)
                starts[tail[0]] = (tail, tail_num)
                ends[tail[-1]] = (tail, tail_num)
        elif tail is None and head is None:
            new = deque((frm, to))
            contours[current] = new
            starts[frm] = (new, current)
            ends[to] = (new, current)
            current += 1
        elif head is None:
            tail.appendleft(frm)
            starts[frm] = (tail, tail_num)
        else:
            head.append(to)
            ends[to] = (head, head_num)
    return [np.array(c) for _, c in sorted(contours.items())]


def find_contours(image, level):
    """skimage.measure.find_contours(image, level) with the default 'low' options: a list of
    float64 [V, 2] (row, col) arrays."""
    return _assemble(_segments(image, level))


def contours_by_cycles(image, level):
    """The same contours for a closed-contour image (every contour closed, e.g. padded): number
    the segments in emission order, follow each segment to the one leaving its to-point, order
    the cycles by their smallest number and start each at the to-point of its largest number."""
    segs = [s for s in _segments(image, level) if s[0] != s[1]]
    leaving = {frm: i for i, (frm, _) in enumerate(segs)}
    assert len(leaving) == len(segs)
    succ = [leaving[to] for _, to in segs]
    seen = [False] * len(segs)
    cycles = []
    for i in range(len(segs)):
        if seen[i]:
            continue
        cyc = [i]
        seen[i] = True
        j = succ[i]
        while j != i:
            cyc.append(j)
            seen[j] = True
            j = succ[j]
        cycles.append(cyc)            # discovered in order of their smallest number
    out = []
    for cyc in cycles:
        assert len(cyc) >= 4
        m = max(cyc)
        verts = [segs[m][1]]
        j = succ[m]
        for _ in range(len(cyc)):
            verts.append(segs[j][1])
            j = succ[j]
        out.append(np.array(verts, dtype=np.float64))
    return out


def mask_polygons(boxes, masks):
    """The polygon loop of display_instances: per instance, a list of float64 [V, 2] (x, y)
    arrays (no contour for an instance whose box is all zeros)."""
    masks = np.asarray(masks)
    H, W = masks.shape[:2]
    out = []
    for i in range(int(np.asarray(boxes).shape[0])):
        if not np.any(boxes[i]):
            out.append([])
            continue
        padded = np.zeros((H + 2, W + 2), dtype=np.uint8)
        padded[1:-1, 1:-1] = masks[:, :, i]
        out.append([np.fliplr(v) - 1 for v in _find_contours_cropped(padded)])
    return out


def _find_contours_cropped(padded):
    """find_contours(padded, 0.5) of a zero-bordered 0/1 image, traced on the smallest window
    holding every set pixel and its ring (the cells outside it emit nothing)."""
    rows, cols = np.nonzero(padded.any(axis=1))[0], np.nonzero(padded.any(axis=0))[0]
    if rows.size == 0:
        return []
    r0, c0 = rows[0] - 1, cols[0] - 1
    win = padded[r0:rows[-1] + 2, c0:cols[-1] + 2]
    return [v + np.array([r0, c0], dtype=np.float64) for v in _assemble(_segments_fast(win, 0.5))]
