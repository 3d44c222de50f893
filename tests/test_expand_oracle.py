"""The restatement of the mask-expand sample (expand_oracle.py) on the CPU: its fmaf is exact, it
stays within the float64 contract with upstream, the floor estimate the kernels correct is known
extent by extent, and each one-line departure from the definition changes what the exact GPU
tests (test_gpu_expand_exact.py) compare, on those tests' own inputs."""
import dataclasses
from fractions import Fraction

import numpy as np
import pytest

import oracle

import expand_inputs as ei
import expand_oracle as eo

MAX_EXTENT = 2048


# ------------------------------------------------------------------------------- fmaf
def _round32(x):
    """float32 nearest to the Fraction x, ties to even; inf past the overflow threshold."""
    with np.errstate(over="ignore"):
        c = np.float32(float(x))                 # within an ulp of the answer
    cands = [c] + [np.nextafter(c, np.float32(s)) for s in (-np.inf, np.inf)]
    cands = [v for v in cands if np.isfinite(v)]
    top = Fraction(2) ** 128 - Fraction(2) ** 103          # FLT_MAX + half an ulp
    if abs(x) >= top:
        return np.float32(np.inf if x > 0 else -np.inf)
    best = min(cands, key=lambda v: (abs(Fraction(float(v)) - x),
                                     int(np.array(v, np.float32).view(np.uint32)) & 1))
    if best == 0:                                # an underflow keeps the sign of the exact value
        return np.float32(-0.0 if x < 0 else 0.0)
    return best


def _fma_exact(a, b, c):
    """fmaf of three finite float32 values, from exact rationals."""
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if exact == 0:
        # IEEE: an exact zero sum is +0 under round to nearest, unless both terms are -0
        prod_neg = (np.signbit(a) != np.signbit(b))
        neg = prod_neg and np.signbit(c) and float(a) * float(b) == 0 and float(c) == 0
        return np.float32(-0.0 if neg else 0.0)
    return _round32(exact)


def _same32(x, y):
    return np.array(x, np.float32).view(np.uint32) == np.array(y, np.float32).view(np.uint32) or \
        (np.isnan(x) and np.isnan(y))


def _double_rounding_cases():
    """Triples whose product is exactly a float32 rounding midpoint M and whose addend is a tiny
    nudge: a * b + c lies just beside M, float64 rounds it onto M, and the float32 cast then
    breaks the tie the wrong way half the time."""
    out = []
    for e in (1, 2, 5, 11):
        a = np.float32(1 + 2.0 ** -12)
        b = np.float32(1 + 2.0 ** -12)               # a * b = 1 + 2^-11 + 2^-24: a midpoint
        for s in (1, -1):
            for nudge in (2.0 ** -80, 2.0 ** -60, 2.0 ** -126, 2.0 ** -149):
                out.append((np.float32(s * a * 2.0 ** e), b, np.float32(s * nudge * 2.0 ** e)))
                out.append((np.float32(s * a * 2.0 ** e), b, np.float32(-s * nudge * 2.0 ** e)))
    return out


def test_fma32_is_exactly_rounded():
    rng = np.random.default_rng(1)
    triples = []
    # random values over a wide exponent range, and near-cancelling sums
    for _ in range(3000):
        a, b, c = (np.float32(rng.standard_normal() * 2.0 ** rng.integers(-40, 40))
                   for _ in range(3))
        triples.append((a, b, c))
        near = -float(a) * float(b) * (1 + rng.integers(-3, 4) * 2.0 ** -24)
        triples.append((a, b, np.float32(near)))
    # subnormal operands and results, signed zeros, overflow
    sub = [np.float32(2.0 ** -149), np.float32(-(2.0 ** -149)), np.float32(3 * 2.0 ** -140),
           np.float32(2.0 ** -126), np.float32(0.0), np.float32(-0.0), np.float32(1.5),
           np.float32(-0.75), np.float32(3e38), np.float32(-3e38), np.float32(2.0 ** 64),
           np.float32(2.0 ** -70), np.float32(2.0 ** -75)]
    triples += [(a, b, c) for a in sub for b in sub for c in sub]
    cases = _double_rounding_cases()
    triples += cases
    a, b, c = (np.array(v, dtype=np.float32) for v in zip(*triples))
    got = eo.fma32(a, b, c)
    for i, t in enumerate(triples):
        want = _fma_exact(*t)
        assert _same32(got[i], want), (t, got[i], want)
    # the naive float64 form double-rounds on the constructed triples: the test above would
    # notice fma32 degrading to it
    a, b, c = (np.array(v, dtype=np.float32) for v in zip(*cases))
    naive = (a.astype(np.float64) * b + c).astype(np.float32)
    wrong = sum(not _same32(naive[i], _fma_exact(*t)) for i, t in enumerate(cases))
    assert wrong > 0


def test_fma32_non_finite_operands():
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    one, zero = np.float32(1), np.float32(0)
    got = eo.fma32([inf, zero, inf, one, one, inf, np.float32(3e38)],
                   [one, inf, one, one, nan, zero, np.float32(2)],
                   [one, one, -inf, inf, one, one, np.float32(3e38)])
    want = [np.inf, np.nan, np.nan, np.inf, np.nan, np.nan, np.inf]
    for g, w in zip(got, want):
        assert (np.isnan(g) and np.isnan(w)) or g == w, (got, want)


# ------------------------------------------------------------------------------- floor estimate
def test_floor_correction_extents():
    """__float2int_rd(fl(A) * fl(1/D)) against the exact floor of A / D for every tile side
    2 .. 64 (MRX_MAX_MASK_DIM) and every extent up to 2048.

    The estimate is never too high there, and it cannot be anywhere the ABI's integers are exact:
    it exceeds A / D by at most |A / D| (2^-23 + 2^-48) (two roundings of 2^-24 each), while a
    quotient below an integer is at least 1 / D below it, so a too-high estimate needs |A| >= 2^23,
    that is an extent above 2^23 / (2 * side) (65536 at side 64, 149796 at side 28).  It is too
    low only where A / D is an exact integer and the product rounds below it, at a few extents per
    side: those run src_floor's correction (rem >= D), which the GPU test drives through
    expand_inputs' `floor` family."""
    per_side = {}
    for side in range(2, 65):
        low, high = eo.floor_estimate_misses(side, MAX_EXTENT)
        assert high.sum() == 0, (side, np.nonzero(high)[0] + 1)
        per_side[side] = eo.floor_correction_extents(side, MAX_EXTENT)
        assert per_side[side] == [int(e) + 1 for e in np.nonzero(low)[0]]
    at28 = per_side[28]
    assert at28 and at28[0] == 244, at28
    # below 2048 every side but 64 has some
    assert all(per_side[s] for s in range(2, 64)) and not per_side[64]
    # the exact integer coordinates where it misses: spot-check one offset of the first extent
    ext = 244
    i, rem = eo.src_floor(28, np.arange(ext), ext)
    A = 28 * (2 * np.arange(ext) + 1) - ext
    est = np.floor(A.astype(np.float32) * (np.float32(1) / np.float32(2 * ext))).astype(np.int64)
    miss = np.nonzero(est != i)[0]
    assert miss.size and (rem[miss] == 0).all() and (est[miss] == i[miss] - 1).all()


# ------------------------------------------------------------------------------- float64 contract
def _extent_pairs(rng, count):
    edge = [1, 2, 3, 27, 28, 29, 56, 244, 1023, 2048]
    pairs = [(h, w) for h in edge for w in (1, 28, 2048) if h * w <= 1 << 21]
    e = np.exp(rng.uniform(0, np.log(MAX_EXTENT), size=(count, 2))).astype(np.int64) + 1
    pairs += [(int(h), int(w)) for h, w in np.minimum(e, MAX_EXTENT) if h * w <= 1 << 21]
    return pairs


@pytest.mark.parametrize("mask_hw", [(28, 28), (33, 12), (64, 64), (2, 4)])
def test_restatement_within_float64_contract(mask_hw):
    """For [0, 1] tiles the definition stays within MASK_VALUE_ATOL = 1e-6 of upstream's float64
    resize at every box extent (a seeded sample of 1 .. 2048 on each axis), which is the
    tolerance the float64 GPU tests assert; at extent == tile side it is the tile itself."""
    rng = np.random.default_rng(sum(mask_hw))
    tile = rng.random(mask_hw)
    worst = 0.0
    for bh, bw in _extent_pairs(rng, 24):
        v = eo.sample(tile, bh, bw)
        ref = oracle.resize(tile.astype(np.float32).astype(np.float64), (bh, bw))
        worst = max(worst, float(np.abs(v.astype(np.float64) - ref).max()))
    assert worst <= 1e-6, worst
    ident = eo.sample(tile, *mask_hw)
    assert np.array_equal(ident.view(np.uint32), tile.astype(np.float32).view(np.uint32))
    assert np.array_equal(ident, oracle.resize(tile.astype(np.float32).astype(np.float64),
                                               mask_hw))


def test_tile_rounds_to_nearest_even():
    t = np.array([[0.5 - 2.0 ** -26, np.nextafter(0.5 - 2.0 ** -26, 0)],
                  [0.5 + 2.0 ** -25, 1e39]])
    got = eo.to_tile32(t)
    assert got[0, 0] == np.float32(0.5) and got[0, 1] == np.float32(0.5 - 2.0 ** -25)
    assert got[1, 0] == np.float32(0.5) and got[1, 1] == np.inf


# ------------------------------------------------------------------------------- discrimination
def test_inputs_give_the_intended_boxes():
    """Every case's boxes survive the normalisation round trip (upstream's box steps)."""
    for f in ei.FAMILIES:
        for p in ei.PATHS:
            im, R, dtype, boxes = ei.case(f, p)
            assert np.array_equal(ei.oracle_boxes(im), boxes), (f, p)
            assert len(boxes) == im.n_valid and im.detections.shape[0] == R


def _differences(variant, need_values):
    """(mask bits, observable values) that differ from the definition over the GPU test's cases,
    stopping at the first family / path that shows what is needed."""
    masks = values = 0
    for f in ei.FAMILIES:
        for p in ei.PATHS:
            im, R, dtype, boxes = ei.case(f, p)
            m0, v0 = ei.restated(im, boxes)
            m1, v1 = ei.restated(im, boxes, variant)
            masks += int((m0 != m1).sum())
            if ei.lane_kernels(p):    # values are observable through the team kernel
                v1 = v1.astype(np.float32)
                same = (v0.view(np.uint32) == v1.view(np.uint32)) | (np.isnan(v0) & np.isnan(v1))
                values += int((~same).sum())
            if masks and (values or not need_values):
                return masks, values
    return masks, values


@pytest.mark.parametrize("name", list(eo.VARIANTS))
def test_each_variant_changes_what_the_gpu_test_compares(name):
    """Each one-line departure from the definition sets or clears at least one mask pixel on the
    exact GPU test's inputs, so every kernel's comparison there can fail; where the departure
    moves a value (all but `strict`) the team kernel's values differ too."""
    masks, values = _differences(eo.VARIANTS[name], need_values=name != "strict")
    assert masks > 0, name
    if name != "strict":
        assert values > 0, name


def test_variants_are_one_change_each():
    assert eo.DEFINITION == eo.Variant()
    for name, v in eo.VARIANTS.items():
        assert sum(dataclasses.asdict(v).values()) == 1 and getattr(v, name)
