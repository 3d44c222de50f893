"""CPU checks of tests/contour_edge_inputs.py: every builder still holds the edges it names (the
census), every input traces to an even segment total, and every closed form the GPU edge tests
compare against equals tests/contour_oracle.py on small sizes."""
import numpy as np
import pytest

import contour_edge_inputs as E
import contour_oracle as co


@pytest.fixture(scope="module")
def built():
    return {name: f() for name, f in E.BUILDERS.items()}


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_builder_holds_its_edges(built, name):
    got = E.census(built[name]["batches"])
    short = {k: (got[k], v) for k, v in built[name]["expect"].items() if got[k] < v}
    assert not short, f"{name}: (found, wanted) {short}"


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_segment_totals_are_even(built, name):
    """Each closed boundary has an even number of unit edges, so S is even; the tile cases are
    stated as even counts for that reason."""
    for b in built[name]["batches"]:
        S = sum(E.cycles(m, r)[0] for _, _, m, r in E.instances(b))
        assert S % 2 == 0, (b["name"], S)


def _flat(polys):
    verts = np.concatenate(polys) if polys else np.zeros((0, 2))
    return verts, np.concatenate([[0], np.cumsum([len(p) for p in polys])]).astype(np.int64)


@pytest.mark.parametrize("H,W", [(1, 1), (1, 6), (5, 1), (4, 4), (5, 7), (8, 9), (13, 12)])
@pytest.mark.parametrize("parity", [0, 1])
def test_checkerboard_closed_form(H, W, parity):
    m = E.checkerboard(H, W, parity)
    want = co.mask_polygons(np.ones((1, 4), np.int32), m[:, :, None])[0]
    verts, off = E.checkerboard_polygons(H, W, parity)
    wv, wo = _flat(want)
    assert np.array_equal(off, wo) and np.array_equal(verts, wv)
    assert np.array_equal((verts, off)[0], E.dots_polygons(m)[0])


@pytest.mark.parametrize("n_seg,width", [(4, 8), (6, 8), (4094, 64), (4096, 66), (16388, 128)])
def test_dots_closed_form(n_seg, width):
    m = E.dots(n_seg, width)
    S, cyc = E.cycles(m, (0, 0) + m.shape)
    assert S == n_seg and sum(L for _, L in cyc) == n_seg
    if n_seg % 4 == 0 and n_seg <= 4096:         # no domino: every pixel a diamond
        want = co.mask_polygons(np.ones((1, 4), np.int32), m[:, :, None])[0]
        verts, off = E.dots_polygons(m)
        wv, wo = _flat(want)
        assert np.array_equal(off, wo) and np.array_equal(verts, wv)


@pytest.mark.parametrize("L", [4, 6, 8, 14, 16, 18, 62, 64, 66, 1022, 1024, 1026])
def test_rectangles_and_snakes_have_one_cycle_of_L(L):
    for h in (1, 3, 17):
        if h < L // 2:
            m = E.rectangle(h, L // 2 - h)
            assert E.cycles(m, (0, 0) + m.shape)[1] == [(0, L)]
    for run in (1, 2, 16, 64, 255):
        m = E.snake((L - 2) // 2, max(1, min(run, (L - 2) // 2)))
        S, cyc = E.cycles(m, (0, 0) + m.shape)
        assert S == L and len(cyc) == 1
        polys = co.mask_polygons(np.ones((1, 4), np.int32), m[:, :, None])[0]
        assert len(polys) == 1 and len(polys[0]) == L + 1


def test_cycles_number_segments_as_the_oracle_orders_contours():
    """`cycles` (the census' numbering) gives one cycle per oracle contour, in the same order, of
    the same length."""
    rng = np.random.default_rng(5)
    for hw in [(7, 9), (20, 33), (40, 70)]:
        m = E.noise(rng, *hw)
        reg = (2, 3, hw[0] - 1, hw[1] - 2)
        S, cyc = E.cycles(m, reg)
        want = E.reference(m, reg)
        assert [L for _, L in cyc] == [len(p) - 1 for p in want]
        assert S == sum(L for _, L in cyc)


@pytest.mark.parametrize("n", [17, 40, 1000])
def test_far_apart_reference(n):
    """The windows' reference equals the oracle on the whole mask, both ways round."""
    row = np.zeros((1, n), bool)
    row[0, [0, 1, 3, n - 5, n - 4, n - 1]] = True
    for mask, blobs in ((row, [(0, 0, 1, 8), (0, n - 8, 1, n)]),
                        (row.T.copy(), [(0, 0, 8, 1), (n - 8, 0, n, 1)])):
        want = co.mask_polygons(np.ones((1, 4), np.int32), mask[:, :, None])[0]
        got = E.far_apart_reference(mask, blobs)
        assert len(got) == len(want) and all(np.array_equal(a, b) for a, b in zip(got, want))


def test_long_masks_lie_past_float32():
    """Case E's coordinates are ones float32 cannot hold: the last vertex of each long mask."""
    for name, mask, blobs in E.long_masks():
        last = E.far_apart_reference(mask, blobs)[-1]
        assert (last.astype(np.float32).astype(np.float64) != last).any(), name


def test_cut_reference_ignores_pixels_outside():
    rng = np.random.default_rng(6)
    m = E.noise(rng, 12, 20)
    for reg in [(-3, 2, 7, 15), (2, -5, 9, 30), (4, 4, 4, 9), (6, 2, 3, 9), (5, 5, 6, 6)]:
        g = E.clamp(reg, 12, 20)
        flipped = m.copy()
        if g is None:
            flipped[:] = ~m
        else:
            y1, x1, y2, x2 = g
            keep = np.zeros_like(m)
            keep[y1:y2, x1:x2] = True
            flipped[~keep] = ~m[~keep]
        a, b = E.reference(m, reg), E.reference(flipped, reg)
        assert len(a) == len(b) and all(np.array_equal(p, q) for p, q in zip(a, b))
