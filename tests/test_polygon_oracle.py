"""The polygon oracle (pycocotools' annToRLE restated) on answers worked by hand from rleFrPoly,
and its properties: the merge is the union of the parts and the runs cover the image."""
import numpy as np
import pytest

import polygon_oracle as po


def test_square():
    """[0,0 10,0 10,10 0,10] on 20 x 20: rows 0-9 x columns 0-9.  The walk's column changes at
    u = 5x + 2 keep x = 0 .. 9 (xd = 10 would need u = 52, past the edge's end at 50); each
    column toggles at yd = 0 (v = 0) and at yd = 10 (v = 50)."""
    m = po.ann_to_mask([[0, 0, 10, 0, 10, 10, 0, 10]], 20, 20)
    want = np.zeros((20, 20), bool)
    want[:10, :10] = True
    assert np.array_equal(m, want)
    assert po.ann_to_rle([[0, 0, 10, 0, 10, 10, 0, 10]], 20, 20) == [0, 10, 10, 10, 10, 10, 10,
                                                                      10, 10, 10, 10, 10, 10, 10,
                                                                      10, 10, 10, 10, 10, 10, 210]


def test_empty_triangle():
    """[0,0 1,1 2,0] on 4 x 6: the kept column changes are at u = 2 -> 3 (x = 0) on the edge up
    and on the base, and at u = 7 -> 8 (x = 1) on the edge down and on the base, all with
    v <= 3, so yd = 0: each column gets two toggles at row 0, they cancel, and the mask is
    empty."""
    assert not po.ann_to_mask([[0, 0, 1, 1, 2, 0]], 4, 6).any()


def test_negative_fraction_truncates():
    """-0.1 scales to (int)(-0.5 + .5) = 0 and -0.15 to (int)(-0.25) = 0 as well, where floor
    would give -1: a vertex a little left of the image behaves as one at 0."""
    a = po.ann_to_mask([[-0.15, -0.1, 6, -0.1, 6, 6, -0.15, 6]], 8, 8)
    b = po.ann_to_mask([[0, 0, 6, 0, 6, 6, 0, 6]], 8, 8)
    assert np.array_equal(a, b) and a.sum() == 36
    assert int(5.0 * -0.15 + .5) == 0 and np.floor(5.0 * -0.15 + .5) == -1


def test_box_list():
    """[x, y, w, h] parts are rleFrBbox's polygons: [2, 3, 4, 5] is columns 2-5 x rows 3-7."""
    m = po.ann_to_mask([[2, 3, 4, 5]], 10, 10)
    want = np.zeros((10, 10), bool)
    want[3:8, 2:6] = True
    assert np.array_equal(m, want)
    with pytest.raises(ValueError):
        po.fr_py_objects([[2, 3, 4, 5], [1, 2, 3, 4, 5, 6]], 10, 10)


def test_odd_length_part():
    """A trailing odd number is dropped: 9 numbers are 4 vertices."""
    assert np.array_equal(po.ann_to_mask([[0, 0, 10, 0, 10, 10, 0, 10, 99]], 20, 20),
                          po.ann_to_mask([[0, 0, 10, 0, 10, 10, 0, 10]], 20, 20))


def test_overlapping_parts_union():
    """Two overlapping squares: the union (an XOR would clear rows 5-9 x columns 5-9)."""
    m = po.ann_to_mask([[0, 0, 10, 0, 10, 10, 0, 10], [5, 5, 15, 5, 15, 15, 5, 15]], 20, 20)
    assert m.sum() == 100 + 100 - 25
    assert m[5:10, 5:10].all()


def test_toggle_at_row_h():
    """A polygon reaching past the bottom: its lower toggles clamp to yd = H, position
    x*H + H = (x+1)*H, which ends the column (no pixel of the next column is set by it)."""
    m = po.ann_to_mask([[3, 0, 3, 40, 6, 40, 6, 0]], 20, 10)
    want = np.zeros((20, 10), bool)
    want[:, 3:6] = True
    assert np.array_equal(m, want)


def test_dispatch_errors():
    for bad in ([], [[1, 2, 3]], [[1, 2]]):
        with pytest.raises(ValueError):
            po.fr_py_objects(bad, 5, 5)


@pytest.mark.parametrize("seed", range(4))
def test_merge_is_union_and_runs_cover(seed):
    rng = np.random.default_rng(seed)
    for _ in range(40):
        H, W = int(rng.integers(1, 30)), int(rng.integers(1, 30))
        parts = [[float(v) for v in rng.uniform(-3, max(H, W) + 3, 2 * int(rng.integers(3, 8)))]
                 for _ in range(int(rng.integers(1, 4)))]
        runs = [po.fr_poly(p, H, W) for p in parts]
        for r in runs:
            assert sum(r) == H * W
        merged = po.merge(runs, H, W)
        assert sum(merged) == H * W
        want = np.zeros((H, W), bool)
        for r in runs:
            want |= po.decode(r, H, W)
        assert np.array_equal(po.decode(merged, H, W), want)
