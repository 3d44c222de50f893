"""CPU restatement of the sample every mask-expand kernel computes, bit for bit.  TEST
INFRASTRUCTURE ONLY.

csrc/expand.cuh defines the sample (DESIGN.md 3.1).  Canvas pixel d of a box [lo, lo + ext)
samples the zero-padded tile (`in` samples on that axis) at the source coordinate A / D,
A = in * (2 (d - lo) + 1) - ext, D = 2 ext:

  - the floor i and remainder rem of A / D are integers;
  - the weight is float32(rem) * fl32(1 / D), the reciprocal rounded to nearest;
  - a lerp is fmaf(w, hi - lo, lo), with hi - lo a float32 subtraction;
  - rows i and i + 1 are interpolated horizontally, then the two results vertically;
  - the pixel is set when the sample is >= 0.5f.

The tile itself is float32: a float64 input is rounded to nearest even (unmold_prepare_kernel's
static_cast<float>), values above FLT_MAX becoming inf.

`fma32` emulates fmaf exactly with float64 arithmetic: the product of two float32 values is exact
in float64, an exact TwoSum with the addend gives the float64 sum and its error, the sum is
rounded to odd from them, and the cast to float32 then rounds once more, correctly because
53 >= 24 + 2.  Rounding a*b + c once in float64 and then to float32 rounds twice and is wrong on
some inputs (test_expand_oracle.py shows one).

`Variant` names the one-line departures from the definition that the kernels could make without
the float64 band tests noticing; the CPU discrimination tests use them to show that the GPU
comparisons can fail.  Everything else uses `DEFINITION`.
"""
import dataclasses
import functools

import numpy as np

import oracle


@dataclasses.dataclass(frozen=True)
class Variant:
    unfused: bool = False          # lerp as a float32 multiply, then an add
    one_minus: bool = False        # lerp as (1 - w) * lo + w * hi
    vertical_first: bool = False   # interpolate the two columns vertically, then horizontally
    div_weight: bool = False       # w = fl(rem / D) instead of rem * fl(1 / D)
    rcp_rz: bool = False           # 1 / D rounded toward zero
    strict: bool = False           # > 0.5 instead of >= 0.5
    f64_tile: bool = False         # the whole sample in float64 from the unrounded tile


DEFINITION = Variant()
VARIANTS = {f.name: Variant(**{f.name: True}) for f in dataclasses.fields(Variant)}


# ------------------------------------------------------------------------------- fmaf
def fma32(a, b, c):
    """float32 fmaf(a, b, c) elementwise: a * b + c rounded once, to nearest even.  Non-finite
    operands take plain float64 evaluation (IEEE's inf and NaN); a finite result past FLT_MAX
    becomes inf on the cast."""
    a, b, c = (np.asarray(x, dtype=np.float32) for x in (a, b, c))
    a, b, c = np.broadcast_arrays(a, b, c)
    with np.errstate(all="ignore"):
        a64, b64, c64 = (x.astype(np.float64) for x in (a, b, c))
        p = a64 * b64                              # exact: 24 + 24 significant bits
        s = p + c64
        bp = s - c64                               # TwoSum (Knuth): s + err == p + c exactly
        err = (p - bp) + (c64 - (s - bp))
        # round to odd: an inexact sum with an even last bit moves one ulp towards the exact value
        even = (s.view(np.int64) & 1) == 0
        odd = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        finite = np.isfinite(a64) & np.isfinite(b64) & np.isfinite(c64)
        out = np.where(finite, odd, p + c64)
        return out.astype(np.float32)


def to_tile32(tile):
    """The float32 tile the kernels read: round to nearest even (inf past FLT_MAX)."""
    with np.errstate(over="ignore"):
        return np.asarray(tile).astype(np.float32)


# ------------------------------------------------------------------------------- source coordinates
def src_floor(in_, d, ext):
    """Exact floor i and remainder rem of A / D for canvas offsets d = 0 .. ext - 1 (int64)."""
    d = np.asarray(d, dtype=np.int64)
    A = int(in_) * (2 * d + 1) - int(ext)
    D = 2 * int(ext)
    i = A // D                                     # floor division, also for A < 0
    return i, A - i * D


def recip32(D, variant=DEFINITION):
    """fl32(1 / D): to nearest (__fdiv_rn), or toward zero (rcp_rz)."""
    r = np.float32(1) / np.float32(D)
    if variant.rcp_rz and float(r) * D > 1.0:      # (exact in float64: 24 x 25 bits)
        r = np.nextafter(r, np.float32(0))
    return np.float32(r)


def axis_weights(in_, ext, variant=DEFINITION):
    """(i, w) of every canvas offset of a box of `ext` pixels on an axis of `in_` tile samples:
    i the exact floor, w the float32 weight (float64 for f64_tile)."""
    i, rem = src_floor(in_, np.arange(int(ext)), ext)
    D = 2 * int(ext)
    if variant.f64_tile:
        return i, rem / D
    if variant.div_weight:
        return i, rem.astype(np.float32) / np.float32(D)
    return i, rem.astype(np.float32) * recip32(D, variant)


def floor_estimate_misses(in_, max_ext):
    """The kernels' estimate of the floor, __float2int_rd(fl32(A) * fl32(1 / D)), against the exact
    floor, for every extent 1 .. max_ext on an axis of `in_` samples.  Returns int64 arrays
    (too_low, too_high): per extent, the number of canvas offsets whose estimate is one below /
    above the floor (index 0 is extent 1)."""
    ext, d = _offset_grid(int(max_ext))
    A = int(in_) * (2 * d + 1) - ext
    D = 2 * ext
    inv = (np.float32(1) / np.arange(2, 2 * max_ext + 1, 2, dtype=np.float32))[ext - 1]
    est = np.floor(A.astype(np.float32) * inv).astype(np.int64)
    exact = A // D
    low = np.bincount(ext[est < exact] - 1, minlength=max_ext)
    high = np.bincount(ext[est > exact] - 1, minlength=max_ext)
    return low, high


@functools.lru_cache(maxsize=2)
def _offset_grid(max_ext):
    """(ext, d) int64 for every extent 1 .. max_ext and every offset d < ext."""
    ext = np.repeat(np.arange(1, max_ext + 1, dtype=np.int64), np.arange(1, max_ext + 1))
    starts = np.repeat(np.cumsum(np.arange(0, max_ext, dtype=np.int64)), np.arange(1, max_ext + 1))
    return ext, np.arange(ext.size, dtype=np.int64) - starts


def floor_correction_extents(in_, max_ext=2048):
    """The extents up to max_ext at which the kernels' floor estimate is off for some offset on an
    axis of `in_` samples: those run src_floor's correction."""
    low, high = floor_estimate_misses(in_, max_ext)
    return [int(e) + 1 for e in np.nonzero(low + high)[0]]


# ------------------------------------------------------------------------------- the sample
def _lerp(w, lo, hi, variant):
    if variant.f64_tile:
        return w * (hi - lo) + lo
    with np.errstate(all="ignore"):
        if variant.unfused:
            return (w * (hi - lo)).astype(np.float32) + lo
        if variant.one_minus:
            return (np.float32(1) - w) * lo + w * hi
        return fma32(w, hi - lo, lo)


def sample(tile, bh, bw, variant=DEFINITION):
    """The pre-threshold samples [bh, bw] of `tile` [mh, mw] resized to a bh x bw box: float32
    (float64 for f64_tile)."""
    tile = np.asarray(tile)
    mh, mw = tile.shape
    t = tile.astype(np.float64) if variant.f64_tile else to_tile32(tile)
    pad = np.zeros((mh + 2, mw + 2), dtype=t.dtype)
    pad[1:-1, 1:-1] = t
    iy, wy = axis_weights(mh, bh, variant)
    ix, wx = axis_weights(mw, bw, variant)
    top, bot = pad[iy + 1], pad[iy + 2]            # [bh, mw + 2]: source rows i, i + 1
    wx, wy = wx[None, :], wy[:, None]
    if variant.vertical_first:
        left = _lerp(wy, top[:, ix + 1], bot[:, ix + 1], variant)
        right = _lerp(wy, top[:, ix + 2], bot[:, ix + 2], variant)
        return _lerp(wx, left, right, variant)
    ht = _lerp(wx, top[:, ix + 1], top[:, ix + 2], variant)
    hb = _lerp(wx, bot[:, ix + 1], bot[:, ix + 2], variant)
    return _lerp(wy, ht, hb, variant)


def threshold(values, variant=DEFINITION):
    with np.errstate(invalid="ignore"):
        return values > 0.5 if variant.strict else values >= 0.5


def instance_mask(tile, bh, bw, variant=DEFINITION):
    return threshold(sample(tile, bh, bw, variant), variant)


# ------------------------------------------------------------------------------- outputs
def expand(hw, boxes, tiles, variant=DEFINITION):
    """The byte canvas of one image: (masks bool [H, W, N], values [H, W, N]) for boxes (y1, x1,
    y2, x2) and tiles [N, mh, mw]; masks are zero and values NaN outside each box."""
    H, W = (int(v) for v in hw)
    n = len(boxes)
    masks = np.zeros((H, W, n), dtype=np.bool_)
    values = np.full((H, W, n), np.nan, dtype=np.float64 if variant.f64_tile else np.float32)
    for k, (y1, x1, y2, x2) in enumerate(np.asarray(boxes, dtype=np.int64).reshape(-1, 4)):
        v = sample(tiles[k], y2 - y1, x2 - x1, variant)
        values[y1:y2, x1:x2, k] = v
        masks[y1:y2, x1:x2, k] = threshold(v, variant)
    return masks, values


def packed(masks):
    """The packed planes uint8 [N, H, ceil(W / 8)] of masks [H, W, N]: np.packbits of each row,
    padding bits zero."""
    return np.packbits(masks.transpose(2, 0, 1), axis=-1)


def rle_runs(masks):
    """The uncompressed COCO run lengths of each of masks [H, W, N] (the encoder behind
    coco_oracle.encode)."""
    return [oracle.rle_encode(masks[:, :, k])["counts"] for k in range(masks.shape[2])]
