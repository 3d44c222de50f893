"""Inputs for the scoring kernels at their ties and bounds, built in NumPy: IoU tables for
mrx_coco_match / mrx_coco_match_f64area and mrx_mask_matches drawn from a few values (every
threshold exactly, one ulp either side, 0, 1 - 1e-10, 1, NaN), packed planes for the pair walk at
every byte alignment, and a box / mask dataset whose IoUs and areas land on the thresholds and the
area bounds.  Each builder is seeded; tests/test_score_edge_oracle.py counts the edges each one
holds, so that an edit cannot drop one silently.  TEST INFRASTRUCTURE ONLY."""
from fractions import Fraction

import numpy as np

import cocoeval_oracle as co
import eval_oracle as eo

MAX_T, MAX_A = 64, 16          # MRX_MAX_IOU_THRESHOLDS, MRX_MAX_AREA_RANGES (checked by the tests)
CAP = 1 - 1e-10                # evaluateImg's min(t, 1 - 1e-10)
COCO_THRS = co.Params().iouThrs
COCO_RNG = [[0.0, 1e10], [0.0, 1024.0], [1024.0, 9216.0], [9216.0, 1e10]]


def ulps(x):
    """x and its float64 neighbours."""
    return [np.nextafter(x, -np.inf), x, np.nextafter(x, np.inf)]


def thresholds64():
    """MAX_T thresholds as the kernels take them (capped): COCO's ten (0.8999999999999999
    among them), 1.0 capped, 0.0, then i/u for growing u, each as its float64 quotient."""
    thr = [min(float(t), CAP) for t in COCO_THRS] + [CAP, 0.0]
    u = 2
    while len(thr) < MAX_T:
        thr += [i / u for i in range(1, u) if i / u not in thr][:MAX_T - len(thr)]
        u += 1
    return thr


def area_ranges16():
    """MAX_A ranges: COCO's four, then ranges whose bounds are the areas' edges (32^2 and 96^2
    again, half-integers, an empty range, a point range, bounds one ulp off)."""
    r = list(COCO_RNG) + [[1024.0, 1024.0], [1023.5, 9216.5], [0.0, 0.0], [1.0, 1023.0],
                          [np.nextafter(1024.0, 0), np.nextafter(9216.0, np.inf)],
                          [np.nextafter(1024.0, np.inf), 9216.0], [50.0, 49.0], [9217.0, 1e10],
                          [0.0, 1.0], [2.0, 2.0], [1025.0, 9215.0], [0.0, 1024.0]]
    return [[float(a), float(b)] for a, b in r[:MAX_A]]


def area_edges(ranges, integer):
    """Every bound of `ranges`, the integers next to it (integer) or its ulp neighbours, and 0."""
    out = {0.0}
    for lo, hi in ranges:
        for v in (lo, hi):
            if v > 1e9:
                continue
            out |= {float(np.floor(v)), float(np.floor(v)) + 1, float(np.ceil(v)) - 1} if integer \
                else set(ulps(v))
    return sorted(x for x in out if x >= 0)


def iou_values(thr):
    """0, every threshold and its ulp neighbours, 1 - 1e-10 and 1."""
    v = {0.0, CAP, 1.0}
    for t in thr:
        v |= {x for x in ulps(t) if 0 <= x <= 1}
    return sorted(v)


# ----------------------------------------------------------------------------- mrx_coco_match
def coco_match_case(seed, ms=(1, 31, 32, 33, 64, 65), n_pred=24, T=MAX_T, A=MAX_A,
                    area_type=np.int64):
    """A batch for mrx_coco_match (area_type int64) or mrx_coco_match_f64area (float64): one
    image per M in `ms` with an empty image (no ground truth, then no prediction) between each
    pair; categories 0-2 interleaved (3: a prediction category without ground truth); every IoU
    from a palette of seven values (0.5, 1 - 1e-10 or 0, three thresholds, an ulp below
    one and above another, 1 or one of `iou_values`), equal maxima planted at (j, j + 32) and
    (j, j + 1), crowds, areas on the range bounds, keep = 0 rows and a shuffled walk."""
    rng = np.random.default_rng(seed)
    thr = thresholds64()[:T]
    ranges = area_ranges16()[:A]
    vals = iou_values(thr)
    layout = []
    for k, m in enumerate(ms):
        layout.append((m, n_pred))
        if k + 1 < len(ms):
            layout.append((0, n_pred // 2) if k % 2 == 0 else (m, 0))
    B, R1, R2 = len(layout), n_pred, max(ms)
    c = {"B": B, "R1": R1, "R2": R2, "thresholds": thr, "area_rng": ranges,
         "iou": np.full((B, R1, R2), 1.0), "pred_counts": np.zeros(B, np.int32),
         "pred_cat": np.full((B, R1), -1, np.int32), "pred_keep": np.zeros((B, R1), np.uint8),
         "walk": np.zeros((B, R1), np.int32), "pred_area": np.zeros((B, R1), area_type),
         "gt_counts": np.zeros(B, np.int32), "gt_cat": np.full((B, R2), -1, np.int32),
         "gt_crowd": np.zeros((B, R2), np.uint8), "gt_area": np.zeros((B, R2)),
         "planted": []}
    gt_edges = area_edges(ranges, False)
    dt_edges = area_edges(ranges, area_type == np.int64)
    for b, (m, n) in enumerate(layout):
        c["gt_counts"][b], c["pred_counts"][b] = m, n
        c["gt_cat"][b, :m] = rng.integers(0, 3, m)
        c["gt_crowd"][b, :m] = rng.random(m) < 0.2
        c["gt_area"][b, :m] = rng.choice(gt_edges, m)
        c["pred_cat"][b, :n] = rng.integers(0, 4, n)
        c["pred_keep"][b, :n] = rng.random(n) > 0.15
        c["walk"][b, :n] = rng.permutation(n)
        c["pred_area"][b, :n] = np.asarray(rng.choice(dt_edges, n)).astype(area_type)
        t3 = rng.choice(thr, 3, replace=False)
        palette = np.r_[[0.5, CAP, 0.0][b % 3], t3, np.nextafter(t3[0], 0),
                        np.nextafter(t3[1], 1), 1.0 if b // 2 % 2 else rng.choice(vals)]
        for i in range(n):
            same = np.nonzero(c["gt_cat"][b, :m] == c["pred_cat"][b, i])[0]
            c["iou"][b, i, same] = rng.choice(palette, same.size)
            top = c["iou"][b, i, same].max() if same.size else 0.0
            for d in (32, 1):      # an equal maximum on a lane 32 apart, and on the next lane
                pairs = [j for j in same if j + d in same]
                if pairs and rng.random() < 0.6:
                    j = int(rng.choice(pairs))
                    c["iou"][b, i, [j, j + d]] = top
                    c["planted"].append((b, i, j, j + d))
    return c


def coco_match_cap_case(area_type=np.int64):
    """R2 = 65534 (the ABI's cap): every instance in one image, the few of the predictions'
    category spread to the last one; the first prediction's equal maxima are at 65501 and 65533,
    so it must take j = 65533 (all 16 bits of j, the last word of the matched set)."""
    R2, R1 = 65534, 4
    c = {"B": 2, "R1": R1, "R2": R2, "thresholds": [0.5, 0.75, CAP], "area_rng": COCO_RNG[:2],
         "iou": np.full((2, R1, R2), 1.0), "pred_counts": np.array([R1, R1], np.int32),
         "pred_cat": np.zeros((2, R1), np.int32), "pred_keep": np.ones((2, R1), np.uint8),
         "walk": np.tile(np.arange(R1, dtype=np.int32), (2, 1)),
         "pred_area": np.full((2, R1), 500, area_type),
         "gt_counts": np.array([R2, 0], np.int32), "gt_cat": np.ones((2, R2), np.int32),
         "gt_crowd": np.zeros((2, R2), np.uint8), "gt_area": np.full((2, R2), 500.0),
         "planted": []}
    same = np.r_[0, 31, 32, 33, np.arange(65470, R2, 3), 65533]
    c["gt_cat"][0, same] = 0
    vals = [0.5, 0.75, np.nextafter(0.75, 0), CAP, 0.6]
    for i in range(R1):
        c["iou"][0, i, same] = [vals[(k + i) % len(vals)] for k in range(same.size)]
    c["iou"][0, 0, [65501, 65533]] = 1.0
    c["planted"].append((0, 0, 65501, 65533))
    return c


def expected_coco_match(c, variant=None):
    """(match [A, T, B, R1], ignore [A, T, B, R1]) from cocoeval_oracle.match_image per
    (image, category): -2 / 2 where the kernel writes nothing (kept out, or past the count)."""
    A, T, B, R1 = len(c["area_rng"]), len(c["thresholds"]), c["B"], c["R1"]
    match = np.full((A, T, B, R1), -2, np.int64)
    ignore = np.full((A, T, B, R1), 2, np.int64)
    for b in range(B):
        n, m = int(c["pred_counts"][b]), int(c["gt_counts"][b])
        walk = c["walk"][b, :n]
        kept = [i for i in walk if c["pred_keep"][b, i]]
        for cat in sorted({int(c["pred_cat"][b, i]) for i in kept}):
            D = [i for i in kept if c["pred_cat"][b, i] == cat]
            G = np.nonzero(c["gt_cat"][b, :m] == cat)[0]
            ious = c["iou"][b][np.ix_(D, G)]
            for a, rg in enumerate(c["area_rng"]):
                gtind, _, dtm, _, dtig = co.match_image(
                    ious, c["gt_crowd"][b, G], c["gt_area"][b, G],
                    c["pred_area"][b, D].astype(np.float64), c["thresholds"], rg,
                    variant=variant)
                where = np.where(dtm >= 0, G[gtind][np.maximum(dtm, 0)] if G.size else 0, -1)
                match[a, :, b, D] = where.T
                ignore[a, :, b, D] = dtig.T
    return match, ignore


# ----------------------------------------------------------------------------- mrx_mask_matches
def f32_values(thr):
    """float32 IoUs: 0, 1, NaN, and each threshold's float32 value with its float32 neighbours."""
    v = {np.float32(0), np.float32(1)}
    for t in thr:
        f = np.float32(t)
        v |= {f, np.nextafter(f, np.float32(0)), np.nextafter(f, np.float32(2))}
    return sorted(x for x in v if 0 <= x <= 1) + [np.float32(np.nan)]


MASK_THRESHOLDS = [0.5, np.float64(0.5), 0.7, np.float64(0.7), np.float64(0.55), 0.75,
                   COCO_THRS[8], float(COCO_THRS[8]), 0.95, 1, 0, np.float64(1.0)]


def mask_match_case(seed, ms=(1, 31, 32, 33, 64, 65), n_pred=40):
    """A batch for mrx_mask_matches: float32 overlaps from f32_values, tied and NaN scores,
    classes 1-3 interleaved, equal maxima at (j, j + 32) and (j, j + 1), empty images between."""
    rng = np.random.default_rng(seed)
    vals = f32_values([float(t) for t in MASK_THRESHOLDS])
    layout = []
    for k, m in enumerate(ms):
        layout.append((m, n_pred))
        if k + 1 < len(ms):
            layout.append((0, 5) if k % 2 == 0 else (m, 0))
    B, R1, R2 = len(layout), n_pred, max(ms)
    c = {"B": B, "R1": R1, "R2": R2, "overlaps": np.full((B, R1, R2), np.float32(0.25)),
         "pred_counts": np.zeros(B, np.int32), "pred_cls": np.zeros((B, R1), np.int32),
         "scores": np.zeros((B, R1), np.float32), "gt_counts": np.zeros(B, np.int32),
         "gt_cls": np.zeros((B, R2), np.int32), "planted": []}
    for b, (m, n) in enumerate(layout):
        c["gt_counts"][b], c["pred_counts"][b] = m, n
        c["gt_cls"][b, :m] = rng.integers(1, 4, m)
        c["pred_cls"][b, :n] = rng.integers(1, 4, n)
        s = rng.choice(np.float32([0.9, 0.5, 0.5, 0.3, np.nan, 0.7]), n)
        c["scores"][b, :n] = s
        palette = rng.choice(len(vals), 7, replace=False)
        ov = np.asarray(vals, np.float32)[rng.choice(palette, (n, m))]
        for i in range(n):
            row = ov[i]
            top = np.nanmax(row) if not np.isnan(row).all() else np.float32(1)
            for d in (32, 1):
                if m > d and rng.random() < 0.6:
                    j = int(rng.integers(0, m - d))
                    row[[j, j + d]] = top
                    c["pred_cls"][b, i] = c["gt_cls"][b, j]
                    c["gt_cls"][b, j + d] = c["gt_cls"][b, j]
                    c["planted"].append((b, i, j, j + d))
            if i % 7 == 3 and m:       # one candidate, float32(0.7) or (0.95): below the float64
                row[:] = np.float32(0.25)                   # threshold, not below the Python one
                j = int(rng.integers(0, m))
                row[j] = np.float32([0.7, 0.95][i % 2])
                c["pred_cls"][b, i] = c["gt_cls"][b, j]
        c["overlaps"][b, :n, :m] = ov
    c["score_threshold"] = float(vals[len(vals) // 2])   # equal to IoUs of the matrix
    return c


def expected_mask_matches(c, t, score_threshold, variant=None):
    """(order [B, R1], pred_match [B, R1], gt_match [B, R2]) of compute_matches' loop at threshold
    t (a Python or NumPy number, compared as NumPy compares it); -2 where nothing is written."""
    B, R1, R2 = c["B"], c["R1"], c["R2"]
    order = np.full((B, R1), -2, np.int64)
    pm = np.full((B, R1), -2, np.int64)
    gm = np.full((B, R2), -2, np.int64)
    for b in range(B):
        n, m = int(c["pred_counts"][b]), int(c["gt_counts"][b])
        o = eo.score_order(c["scores"][b, :n], variant)
        order[b, :n] = o
        g, p = eo.match_loop(c["overlaps"][b, o, :m], c["pred_cls"][b, o], c["gt_cls"][b, :m],
                             t, score_threshold, variant)
        pm[b, :n], gm[b, :m] = p, g
    return order, pm, gm


# ----------------------------------------------------------------------------- packed planes
# (H, W): ceil(W/8) % 4 = 0, 1, 2, 3, and H * ceil(W/8) odd where ceil(W/8) is odd
PLANE_SHAPES = [(13, 61), (9, 69), (11, 80), (7, 85), (5, 7), (17, 200)]


def _rect_masks(rng, H, W, n):
    """n masks: rectangles starting and ending at every x & 7, filled at random; one empty, one
    a single column, one a single row, one touching the previous one's right edge, one holding
    the last pixel (the slot's last byte)."""
    out = []
    for k in range(n):
        m = np.zeros((H, W), bool)
        x1 = min((k % 8) + 8 * int(rng.integers(0, max(W // 8, 1))), W - 1)
        x2 = min(x1 + 1 + ((k // 8) % 8) + 8 * int(rng.integers(0, 3)), W)
        y1 = int(rng.integers(0, H))
        y2 = int(rng.integers(y1 + 1, H + 1))
        if k == 1:
            x2 = x1 + 1                               # one pixel wide
        elif k == 2:
            y2 = y1 + 1                               # one pixel high
        elif k == 3 and out[-1].any():
            xs = np.nonzero(out[-1].any(0))[0]
            x1 = min(int(xs[-1]) + 1, W - 1)          # touches without overlapping
            x2 = min(x1 + 5, W)
        m[y1:y2, x1:x2] = rng.random((y2 - y1, x2 - x1)) < 0.75
        m[y1, x1] = m[y2 - 1, x2 - 1] = True
        if k == 4:
            m[H - 1, W - 1] = True                    # the slot's last byte
        if k == 0:
            m[:] = False                              # empty
        out.append(m)
    return out


def extents(m):
    """(y1, x1, y2, x2) exclusive of a mask's set pixels, (0, 0, 0, 0) when empty."""
    if not m.any():
        return (0, 0, 0, 0)
    ys, xs = np.nonzero(m.any(1))[0], np.nonzero(m.any(0))[0]
    return (int(ys[0]), int(xs[0]), int(ys[-1]) + 1, int(xs[-1]) + 1)


def planes_case(seed, n1=20, n2=18):
    """Per image of PLANE_SHAPES: predictions and ground truth as _rect_masks plus copies and
    shifted copies of each other, boundary planes inside each mask's extents, categories,
    crowds and keep flags."""
    rng = np.random.default_rng(seed)
    imgs = []
    for H, W in PLANE_SHAPES:
        gt = _rect_masks(rng, H, W, n2)
        pred = _rect_masks(rng, H, W, n1 - 4) + [gt[5].copy(), gt[6].copy(),
                                                 np.roll(gt[7], 1, axis=1), gt[0].copy()]
        bnd = []
        for m in pred + gt:
            y1, x1, y2, x2 = extents(m)
            q = np.zeros_like(m)
            q[y1:y2, x1:x2] = rng.random((y2 - y1, x2 - x1)) < 0.5
            bnd.append(q)
        imgs.append({"H": H, "W": W, "pred": pred, "gt": gt, "pred_bnd": bnd[:len(pred)],
                     "gt_bnd": bnd[len(pred):], "pred_cat": rng.integers(0, 2, len(pred)),
                     "pred_keep": rng.random(len(pred)) > 0.1,
                     "gt_cat": rng.integers(0, 2, len(gt)), "gt_crowd": rng.random(len(gt)) < 0.3})
    return imgs


def pack_slots(imgs, key, R, lead):
    """uint8 buffer of every image's planes (np.packbits rows, [R, H, ceil(W/8)] per image) at
    slot offsets that start one byte later each image after `lead` bytes, so the planes' bases
    fall at every address mod 4; and the int64 offsets."""
    parts, offs, pos = [], [], 0
    for b, im in enumerate(imgs):
        pad = (lead + b - pos) % 4 + 4
        parts.append(np.zeros(pad, np.uint8))
        pos += pad
        offs.append(pos)
        H, W = im["H"], im["W"]
        planes = np.zeros((R, H, (W + 7) // 8), np.uint8)
        for k, m in enumerate(im[key]):
            planes[k] = np.packbits(m, axis=1)
        parts.append(planes.ravel())
        pos += planes.size
    parts.append(np.zeros(8, np.uint8))
    return np.concatenate(parts), np.asarray(offs, np.int64)


PAIR_VARIANTS = ("first_byte", "last_byte", "crowd_union_gt")


def pair_counts(m1, m2, variant=None):
    """The exact intersection count of two masks; "first_byte" / "last_byte" model and_count
    dropping column x1 of the extents' intersection (unless x1 & 7 == 7, where its first-byte
    mask still covers it) / column x2 - 1."""
    inter = m1 & m2
    n = int(np.count_nonzero(inter))
    if variant in ("first_byte", "last_byte") and n:
        a, b = extents(m1), extents(m2)
        x1, x2 = max(a[1], b[1]), min(a[3], b[3])
        y1, y2 = max(a[0], b[0]), min(a[2], b[2])
        if variant == "first_byte" and x1 & 7 != 7:
            n -= int(np.count_nonzero(inter[y1:y2, x1]))
        if variant == "last_byte":
            n -= int(np.count_nonzero(inter[y1:y2, x2 - 1]))
    return n


def rle_iou_counts(inter, a1, a2, crowd, variant=None):
    """rleIou from exact counts: 0 without intersection, float64 i / u, u = a1 (crowd; a2 under
    "crowd_union_gt") or a1 + a2 - i."""
    if inter == 0:
        return 0.0
    u = (a2 if variant == "crowd_union_gt" else a1) if crowd else a1 + a2 - inter
    return float(inter) / float(u)


def f32_iou(inter, a1, a2):
    """compute_overlaps_masks' float32 order: i / ((a1 + a2) - i), 0 / 0 = NaN."""
    i = np.float32(inter)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.float32(i / np.float32(np.float32(np.float32(a1) + np.float32(a2)) - i))


# ----------------------------------------------------------------------------- boxes and masks
def fma_union(da, g2, g3):
    """da + g2 * g3 rounded once (the contracted union of the box-IoU mutant)."""
    return float(Fraction(da) + Fraction(g2) * Fraction(g3))


def box_dataset():
    """COCO images of boxes (and masks of the integer ones) whose IoUs fall exactly on every
    default threshold and whose w * h and areas fall on 32^2 and 96^2 (and one ulp off), with
    touching, zero-size and negative-size boxes, forty identical instances (equal IoUs on lanes
    j, j + 1 and j + 32), a crowd several detections match, tied scores, two categories
    interleaved and an image without ground truth between full ones.

    Returns (image ids, shapes {id: (H, W)}, gts, dts) with gts dicts {image_id, category_id,
    bbox, area, iscrowd, mask} and dts {image_id, category_id, bbox, score, mask} (mask None
    where the box is not an integer one inside the image)."""
    gts, dts = [], []
    shapes = {1: (24, 120), 2: (40, 40), 3: (16, 16), 4: (110, 200), 5: (30, 60)}

    def mask_of(img, bb):
        H, W = shapes[img]
        x, y, w, h = bb
        if not all(float(v).is_integer() for v in bb) or w <= 0 or h <= 0 or x + w > W or \
                y + h > H or x < 0 or y < 0:
            return None
        m = np.zeros((H, W), bool)
        m[int(y):int(y + h), int(x):int(x + w)] = True
        return m

    def gt(img, cat, bb, area=None, crowd=0):
        gts.append({"image_id": img, "category_id": cat, "bbox": [float(v) for v in bb],
                    "area": float(bb[2] * bb[3] if area is None else area), "iscrowd": crowd,
                    "mask": mask_of(img, bb)})

    def dt(img, cat, bb, score):
        dts.append({"image_id": img, "category_id": cat, "bbox": [float(v) for v in bb],
                    "score": float(score), "mask": mask_of(img, bb)})

    # image 1: a 20 x 1 instance per x offset; detections k x 1 give IoU k / 20 for k = 10..20:
    # exactly 0.5, 0.55, ..., 0.95 (and 18/20 just above 0.8999999999999999)
    for r, k in enumerate(range(10, 21)):
        gt(1, 7, [5 * r % 100, r % 20, 20, 1])
        dt(1, 7, [5 * r % 100, r % 20, k, 1], 0.5 + 0.01 * (r % 3))
        dt(1, 7, [5 * r % 100 + 20, r % 20, 3, 1], 0.5)            # touches: IoU 0
    dt(1, 7, [3, 3, 0, 5], 0.9)                                     # zero width
    dt(1, 7, [8, 2, -3, 4], 0.9)                                    # negative width, area -12
    dt(1, 8, [0, 0, 5, -2], 0.4)                                    # negative height
    gt(1, 8, [0, 0, 10, 10], area=0.0)
    gt(1, 8, [50, 5, -2, 3])                                        # negative width
    # image 2: forty identical instances, ten of them ignored by area; detections equal to them
    for j in range(40):
        gt(2, 7, [4, 4, 16, 16], area=[1024.0, 300.0, np.nextafter(1024.0, 0)][j % 3] if j % 4
           else 9216.0)
    for i in range(30):
        dt(2, 7, [4, 4, 16, 16], 0.7 if i % 2 else 0.6)
    dt(2, 7, [4, 4, 16, 8], 0.6)                                    # IoU exactly 0.5
    # image 3: no ground truth, detections of both categories
    dt(3, 7, [0, 0, 8, 8], 0.8)
    dt(3, 8, [1, 1, 4, 4], 0.8)
    # image 4: w * h on 32^2 and 96^2, one ulp either side, and a crowd region
    gt(4, 8, [0, 0, 200, 110], crowd=1)
    for bb, s in (([0, 0, 32, 32], .9), ([40, 0, 64, 144], .9), ([110, 0, 96, 96], .8),
                  ([0, 40, 32, np.nextafter(32.0, np.inf)], .8), ([0, 80, 32, 31.999], .7),
                  ([150, 50, 48, 48], .7), ([60, 60, 32, 32], .6)):
        dt(4, 8, bb, s)
    gt(4, 8, [0, 0, 32, 32])
    gt(4, 8, [110, 0, 96, 96], area=9216.0)
    gt(4, 8, [60, 60, 32, 32], area=np.nextafter(9216.0, np.inf))
    # image 5: a crowd that several detections lie inside, with a plain instance over it
    gt(5, 7, [0, 0, 40, 20], crowd=1, area=800.0)
    gt(5, 7, [0, 0, 20, 20], area=1024.0)
    for i, bb in enumerate(([0, 0, 20, 20], [0, 0, 10, 20], [20, 0, 20, 20], [0, 0, 40, 20],
                            [5, 5, 10, 10])):
        dt(5, 7, bb, 0.5 if i < 3 else 0.9)
    # image 6: boxes as results give them (two decimals), where w * h and da + ga - i round
    rng = np.random.default_rng(6)
    shapes[6] = (64, 64)
    for k in range(8):
        x, y = np.round(rng.random(2) * 20, 2)
        w, h = np.round(rng.random(2) * 30 + 5, 2)
        gt(6, 7 + k % 2, [x, y, w, h])
        for s in range(3):
            dx, dy, dw, dh = np.round(rng.normal(0, 1.5, 4), 2)
            dt(6, 7 + k % 2, [x + dx, y + dy, w + dw, h + dh], np.round(rng.random(), 1))
    return [1, 2, 3, 4, 5, 6], shapes, gts, dts
