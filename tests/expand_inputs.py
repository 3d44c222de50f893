"""Seeded inputs of the exact mask-expand tests (test_gpu_expand_exact.py) and of the CPU tests
that show those comparisons can fail (test_expand_oracle.py).  TEST INFRASTRUCTURE ONLY.

A case is one image whose molded shape is its original shape, so that every box is an exact
pixel box: `case(family, path)` gives (SynthImage, R, mask dtype, the intended boxes).  Kept
instance k is detection row k, and its tile is channel class_id of that row.

Families are tile values:
  near       0.5 + k ulp, k in [-8, 8]
  dyadic     {0, 0.25, 0.5, 0.75, 1} at extents tile side x {1/4, 1/2, 1, 2, 4}; instance 0 is a
             constant 0.5 tile
  floor      the extents at which the kernels' fp32 floor estimate is one too low (src_floor's
             correction runs), tiles mixing near-0.5 and small values so that hi - lo is inexact
  f64tie     float64 tiles near 0.5 - 2^-26 and 0.5 + 2^-25, which round onto 0.5 in float32
  subnormal  float32 subnormals, +-0, FLT_MIN, and some 0.5 and 1
  nonfinite  +-inf, NaN, float64 +-1e39, float32 +-3e38 neighbours whose difference overflows
Paths are canvas shapes, tile shapes, R and box heights that steer the kernels (see PATHS).
"""
import numpy as np

import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import synth

import expand_oracle as eo

CLASSES = 3
F32_HALF_ULP_BELOW = 2.0 ** -25      # ulp of float32 just below 0.5
F32_ULP_ABOVE = 2.0 ** -24           # ulp of float32 at 0.5 and above

# name: canvas (H, W), tile (mh, mw), detection rows R, kept instances n, box heights (lo, hi)
# or "full" (y1 = 0, y2 = H), or None (any height up to the canvas)
PATHS = {
    # team kernel, W * N a multiple of 16: every tile row 16-byte aligned (and whole packed words)
    "team_aligned": ((256, 320), (28, 28), 32, 24, None),
    # team kernel, W = 1333 and a ragged N: head / tail bytes, packed rows not word aligned
    "team_unaligned": ((200, 1333), (28, 28), 19, 19, None),
    # team kernel's six-row queue: a full 10-row tile meets more than four source rows
    "team_deep": ((240, 336), (28, 28), 24, 24, (51, 84)),
    # team kernel's general path: one tile meets more than six source rows, boxes below 1.8 sides
    "team_general": ((240, 336), (28, 28), 24, 24, (1, 50)),
    # more boxes than one cull pass holds (128)
    "team_cull_passes": ((160, 480), (28, 28), 160, 150, None),
    # the generic kernel: R above the team limit, or tiles wider than 30 columns
    "generic_R": ((240, 333), (28, 28), 320, 24, None),
    "generic_mw32": ((240, 333), (28, 32), 20, 20, None),
    "generic_mw64": ((200, 256), (20, 64), 20, 20, None),
    # tile shapes with mh != mw
    "tile_28x4": ((240, 333), (28, 4), 20, 20, None),
    "tile_33x28": ((240, 333), (33, 28), 20, 20, None),
    "tile_12x28": ((240, 336), (12, 28), 20, 20, None),
    # full-height boxes: the RLE walk's column-seam sample
    "rle_full_height": ((180, 400), (28, 28), 16, 16, "full"),
}
FAMILIES = ("near", "dyadic", "floor", "f64tie", "subnormal", "nonfinite")
LANE_MASK_W = 30          # MRX_MAX_LANE_MASK_W: the team, bit-packed and RLE kernels
FLOOR_BOXES = 12          # boxes of the floor family that get a listed extent (the rest: small)


def near_values(rng, shape):
    k = rng.integers(-8, 9, size=shape)
    return np.where(k < 0, 0.5 + k * F32_HALF_ULP_BELOW, 0.5 + k * F32_ULP_ABOVE)


def _tiles(family, rng, n, mh, mw):
    """(tiles [n, mh, mw], mask dtype) of a family."""
    shape = (n, mh, mw)
    if family == "near":
        return near_values(rng, shape).astype(np.float32), np.float32
    if family == "dyadic":
        t = rng.choice(np.array([0.0, 0.25, 0.5, 0.75, 1.0]), size=shape)
        t[0] = 0.5
        return t.astype(np.float32), np.float32
    if family == "floor":
        small = rng.random(shape) * 2.0 ** -rng.integers(8, 20, size=shape)
        t = np.where(rng.random(shape) < 0.5, near_values(rng, shape), small)
        return t.astype(np.float32), np.float32
    if family == "f64tie":
        lo, hi = 0.5 - 2.0 ** -26, 0.5 + 2.0 ** -25
        vals = np.array([lo, np.nextafter(lo, 0), np.nextafter(lo, 1), hi, np.nextafter(hi, 0),
                         np.nextafter(hi, 1), 0.5, 0.5 - 2.0 ** -25, 0.0, 1.0])
        return rng.choice(vals, size=shape), np.float64
    if family == "subnormal":
        sub = rng.integers(1, 1 << 23, size=shape).astype(np.uint32).view(np.float32)
        vals = np.where(rng.random(shape) < 0.5, sub, -sub)
        pick = rng.integers(0, 8, size=shape)
        special = np.array([0.0, -0.0, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -126, 0.5, 1.0, 0.0],
                           dtype=np.float32)
        return np.where(pick < 4, vals, special[pick]).astype(np.float32), np.float32
    if family == "nonfinite":
        big = float(np.float32(3e38))
        vals = np.array([np.inf, -np.inf, np.nan, 1e39, -1e39, big, -big,
                         float(np.nextafter(np.float32(big), np.float32(np.inf))), -big * 0.999,
                         0.5, 0.25, 1.0, 0.0, 0.75])
        t = rng.choice(vals, size=shape)
        t[:, :, : mw // 2] = np.where(rng.random((n, mh, mw // 2)) < 0.7, near_values(
            rng, (n, mh, mw // 2)), t[:, :, : mw // 2])
        return t, np.float64
    raise ValueError(family)


def _extents(rng, n, lo, hi, prefer=()):
    """n extents in [lo, hi]; each taken from `prefer` (those inside [lo, hi]) half the time."""
    e = rng.integers(lo, hi + 1, size=n)
    ok = [p for p in prefer if lo <= p <= hi]
    if ok:
        take = rng.random(n) < 0.5
        e[take] = rng.choice(ok, size=int(take.sum()))
    return e


def _boxes(rng, hw, heights, widths, full):
    H, W = hw
    y1 = np.zeros_like(heights) if full else (rng.random(heights.size) * (H - heights + 1)).astype(
        np.int64)
    x1 = (rng.random(widths.size) * (W - widths + 1)).astype(np.int64)
    return np.stack([y1, x1, y1 + heights, x1 + widths], axis=1)


def case(family, path, seed=0):
    """(SynthImage, R, mask dtype, boxes int [n, 4]) of one family on one path."""
    (H, W), (mh, mw), R, n, hrange = PATHS[path]
    rng = np.random.default_rng(_seed(family, path, seed))
    if family == "floor" and R <= 64:
        # room for the listed extents (244, 436, ... at 28 samples), same row alignment as the path
        if hrange is None:
            H = 1000
        W = 1344 if W % 16 == 0 else (1333 if W == 1333 else 1331)
    full = hrange == "full"
    hlo, hhi = (H, H) if full else (hrange or (1, H))
    hpref, wpref = [], []
    if family == "dyadic":
        hpref = [mh * 2 ** k // 4 for k in range(5) if (mh * 2 ** k) % 4 == 0]
        wpref = [mw * 2 ** k // 4 for k in range(5) if (mw * 2 ** k) % 4 == 0]
    heights = _extents(rng, n, hlo, hhi, hpref)
    widths = _extents(rng, n, 1, W, wpref)
    if family != "floor":
        heights = np.minimum(heights, max(hlo, 120))
        widths = np.minimum(widths, 160)
    else:
        # a few boxes with the listed extents, the rest small
        fh = eo.floor_correction_extents(mh, 2048)
        fw = eo.floor_correction_extents(mw, 2048)
        heights = np.minimum(heights, max(hlo, 60))
        widths = np.minimum(widths, 60)
        m = min(n, FLOOR_BOXES)
        ok_h = [e for e in fh if hlo <= e <= hhi]
        ok_w = [e for e in fw if e <= W]
        if ok_h:
            heights[:m] = [ok_h[i % len(ok_h)] for i in range(m)]
        if ok_w:
            widths[:m] = [ok_w[(i + m // 2) % len(ok_w)] for i in range(m)]
    boxes = _boxes(rng, (H, W), heights, widths, full)
    tiles, dtype = _tiles(family, rng, n, mh, mw)
    return make_image((H, W), boxes, tiles, R), R, dtype, boxes


def _seed(family, path, seed):
    return 1000 * (FAMILIES.index(family) + 1) + 10 * list(PATHS).index(path) + seed


def make_image(hw, boxes, tiles, R):
    """A SynthImage whose molded shape is its original shape, with exact pixel boxes; row k keeps
    tile k in channel class_id (1 or 2), the other channels hold 0.75 (a gather of the wrong
    channel shows); rows n .. R - 1 are class-0 padding."""
    H, W = hw
    n, mh, mw = tiles.shape
    det = np.zeros((R, 6), dtype=np.float32)
    det[:n, :4] = synth._norm_boxes_f32(np.asarray(boxes, dtype=np.float64), (H, W))
    cls = 1 + np.arange(n) % 2
    det[:n, 4] = cls
    det[:n, 5] = np.linspace(0.99, 0.7, n)
    msk = np.full((R, mh, mw, CLASSES), 0.75, dtype=tiles.dtype)
    msk[np.arange(n), :, :, cls] = tiles
    return synth.SynthImage(det, msk, (H, W, 3), (H, W, 3), (0, 0, H, W), n)


def oracle_boxes(im):
    """The boxes upstream's unmold_detections computes for `im` (its box steps alone, float64)."""
    det = im.detections.astype(np.float64)
    n = im.n_valid
    window = oracle.norm_boxes(np.array(im.window), im.image_shape[:2])
    wy1, wx1, wy2, wx2 = window
    shift = np.array([wy1, wx1, wy1, wx1])
    scale = np.array([wy2 - wy1, wx2 - wx1, wy2 - wy1, wx2 - wx1])
    return oracle.denorm_boxes((det[:n, :4] - shift) / scale, im.original_image_shape[:2])


def kept_tiles(im):
    """tiles [n, mh, mw] of the kept instances, in the input dtype (row k, channel class_id)."""
    n = im.n_valid
    cls = im.detections[:n, 4].astype(np.int64)
    return im.mrcnn_mask[np.arange(n), :, :, cls]


def restated(im, boxes, variant=eo.DEFINITION):
    """(masks, values) of the image's kept instances, as expand.cuh defines them."""
    return eo.expand(im.original_image_shape[:2], boxes, kept_tiles(im), variant)


def lane_kernels(path):
    """True when the tile shape fits the lane kernels (team, bit-packed, RLE)."""
    return PATHS[path][1][1] <= LANE_MASK_W
