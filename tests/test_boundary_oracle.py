"""CPU tests of the Boundary IoU restatement (tests/boundary_cocoeval_oracle.py): the closed form
of mask_to_boundary (a square erosion with the outside of the image as 0, the rule the device
kernel implements) equals the real cv2 route, and known answers."""
import numpy as np
import pytest

import boundary_cocoeval_oracle as bo


def _random_mask(rng, h, w):
    kind = rng.integers(4)
    if kind == 0:                       # noise of some density
        return rng.random((h, w)) < rng.uniform(0.3, 0.98)
    m = np.zeros((h, w), bool)
    for _ in range(rng.integers(1, 4)):  # rectangles, often touching the edges
        y1, x1 = rng.integers(-3, h), rng.integers(-3, w)
        m[max(y1, 0):max(y1 + rng.integers(1, h + 4), 0), max(x1, 0):max(x1 + rng.integers(1, w + 4), 0)] = True
    if kind == 2:
        m &= rng.random((h, w)) < 0.995  # a few holes
    if kind == 3:
        m[:] = True
    return m


def test_closed_form_equals_cv2():
    rng = np.random.default_rng(5)
    for _ in range(300):
        h, w = (int(v) for v in rng.integers(1, 90, size=2))
        ratio = float(rng.uniform(0.02, 0.3))
        m = _random_mask(rng, h, w)
        d = bo.dilation_of(h, w, ratio)
        want = bo.mask_to_boundary(m, ratio).astype(bool)
        assert np.array_equal(bo.closed_form_boundary(m, d), want), (h, w, ratio, d)


def test_rectangle_is_a_ring():
    h, w = 100, 120
    m = np.zeros((h, w), bool)
    m[20:70, 30:100] = True
    d = bo.dilation_of(h, w)               # round(0.02 * 156.2) = 3
    assert d == 3
    ring = m.copy()
    ring[23:67, 33:97] = False
    assert np.array_equal(bo.mask_to_boundary(m).astype(bool), ring)


def test_edges_keep_a_strip():
    h, w = 60, 80                          # d = 2
    m = np.ones((h, w), bool)
    d = bo.dilation_of(h, w)
    assert d == 2
    want = np.ones((h, w), bool)
    want[d:h - d, d:w - d] = False
    assert np.array_equal(bo.mask_to_boundary(m).astype(bool), want)
    half = np.zeros((h, w), bool)
    half[:, :40] = True                    # touches the top, bottom and left edges
    want = half.copy()
    want[d:h - d, d:40 - d] = False
    assert np.array_equal(bo.mask_to_boundary(half).astype(bool), want)


@pytest.mark.parametrize("h,w,ratio", [(10, 10, 0.5), (3, 40, 0.1), (1, 1, 0.02), (7, 2, 0.3)])
def test_large_dilation_keeps_the_mask(h, w, ratio):
    rng = np.random.default_rng(h * w)
    m = rng.random((h, w)) < 0.9
    assert bo.dilation_of(h, w, ratio) * 2 + 1 > min(h, w)
    assert np.array_equal(bo.mask_to_boundary(m, ratio).astype(bool), m)


@pytest.mark.parametrize("h,w,d", [(1024, 1024, 29), (640, 480, 16), (480, 640, 16),
                                   (800, 1333, 31), (2160, 3840, 88), (5, 5, 1)])
def test_dilation_known_answers(h, w, d):
    assert bo.dilation_of(h, w) == d
