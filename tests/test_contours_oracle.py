"""CPU tests of the contour restatement (tests/contour_oracle.py) and of the host-side checks of
mrx_contours_count / mrx_contours_write: known answers, the closed form the device implements
against the restated `_assemble_contours`, an independent point-in-polygon check, and argument
validation through the library."""
import ctypes as C

import numpy as np
import pytest

import contour_oracle as co
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N


def _polys(mask):
    mask = np.asarray(mask, dtype=bool)
    H, W = mask.shape
    return co.mask_polygons(np.array([[0, 0, H, W]]), mask[:, :, None])[0]


def _xy(pts):
    return np.array(pts, dtype=np.float64)


DIAMOND = _xy([(0, .5), (-.5, 0), (0, -.5), (.5, 0), (0, .5)])


def test_single_pixel():
    got = _polys([[1]])
    assert len(got) == 1 and got[0].dtype == np.float64
    assert np.array_equal(got[0], DIAMOND)


def test_diagonal_pixels_are_two_contours():
    got = _polys([[1, 0], [0, 1]])
    assert len(got) == 2
    assert np.array_equal(got[0], DIAMOND)
    assert np.array_equal(got[1], _xy([(1, 1.5), (.5, 1), (1, .5), (1.5, 1), (1, 1.5)]))


def test_ring_outer_then_hole():
    ring = np.ones((3, 3), bool)
    ring[1, 1] = False
    got = _polys(ring)
    assert len(got) == 2
    assert got[0].shape == (13, 2) and tuple(got[0][0]) == (2, 2.5) and tuple(got[0][-1]) == (2, 2.5)
    assert np.array_equal(got[1], _xy([(1.5, 1), (1, .5), (.5, 1), (1, 1.5), (1.5, 1)]))


def test_all_zero_box_and_empty_mask():
    m = np.ones((4, 5, 2), bool)
    m[:, :, 1] = False
    got = co.mask_polygons(np.array([[0, 0, 0, 0], [0, 0, 4, 5]]), m)
    assert got == [[], []]


def _random_masks(seed, count):
    """Noise, upsampled tiles and dilated specks, padded like display_instances does."""
    from scipy import ndimage

    rng = np.random.default_rng(seed)
    out = []
    for i in range(count):
        h, w = int(rng.integers(1, 24)), int(rng.integers(1, 24))
        kind = i % 3
        if kind == 0:
            m = rng.random((h, w)) < rng.uniform(0.2, 0.8)
        elif kind == 1:
            t = rng.random((int(rng.integers(2, 6)), int(rng.integers(2, 6))))
            m = ndimage.zoom(t, (h / t.shape[0], w / t.shape[1]), order=1) > 0.5
        else:
            m = ndimage.binary_dilation(rng.random((h, w)) < 0.05,
                                        iterations=int(rng.integers(1, 3)))
        p = np.zeros((m.shape[0] + 2, m.shape[1] + 2), np.uint8)
        p[1:-1, 1:-1] = m
        out.append(p)
    return out


def test_fast_segments_equal_the_literal_pass():
    for p in _random_masks(3, 40):
        assert co._segments_fast(p, 0.5) == co._segments(p, 0.5)
    g = np.random.default_rng(4).random((9, 11))          # not only 0/1 images
    assert co._segments_fast(g, 0.4) == co._segments(g, 0.4)


def test_cycle_form_equals_assemble_contours():
    """The closed form the kernels compute (order by the smallest segment number, start at the
    to-point of the largest, follow the successors) equals the dictionary merges."""
    n = 0
    for p in _random_masks(5, 150):
        want = co.find_contours(p, 0.5)
        got = co.contours_by_cycles(p, 0.5)
        assert len(got) == len(want)
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
        n += len(want)
    assert n > 500


def _inside(polys, x, y):
    """Even-odd rule: does the point lie inside the union of the polygons (counted by parity)?"""
    c = False
    for v in polys:
        x0, y0 = v[:-1, 0], v[:-1, 1]
        x1, y1 = v[1:, 0], v[1:, 1]
        cross = (y0 > y) != (y1 > y)
        with np.errstate(divide="ignore", invalid="ignore"):
            xs = x0 + (y - y0) * (x1 - x0) / (y1 - y0)
        c ^= bool(np.count_nonzero(cross & (x < xs)) & 1)
    return c


def test_polygons_reproduce_the_mask():
    """Independent of the restatement's order: every contour is closed, and an even-odd test of
    every pixel centre against an instance's contours gives back its mask (vertices are edge
    midpoints, so no centre lies on an edge)."""
    for p in _random_masks(7, 60):
        m = p[1:-1, 1:-1].astype(bool)
        polys = _polys(m)
        for v in polys:
            assert np.array_equal(v[0], v[-1]) and v.shape[0] >= 5
        got = np.array([[_inside(polys, x, y) for x in range(m.shape[1])]
                        for y in range(m.shape[0])])
        assert np.array_equal(got, m)


def test_contour_entry_points_validate_arguments():
    lib = N.load()
    p16 = C.c_void_p(16)
    assert lib.mrx_contours_count(None, None, None, None, None, None, None, 1, 4, 8, None) == -1
    # mask planes without a region argument
    assert lib.mrx_contours_count(p16, p16, p16, p16, None, p16, p16, 1, 4, 8, None) == -1
    assert b"region" in lib.mrx_last_error()
    assert lib.mrx_contours_count(p16, p16, p16, p16, p16, p16, p16, 1, 0, 8, None) == -1   # R
    args = (p16, p16, p16, p16, p16, p16, p16)
    assert lib.mrx_contours_write(*args, C.c_longlong(10), C.c_longlong(4), p16, p16, None, p16,
                                  1, 4, 8, None) == -1
    assert lib.mrx_contours_write(*args[:4], None, *args[5:], C.c_longlong(10), C.c_longlong(4),
                                  p16, p16, p16, p16, 1, 4, 8, None) == -1
    assert lib.mrx_contours_write(*args, C.c_longlong(10), C.c_longlong(11), p16, p16, p16, p16,
                                  1, 4, 8, None) == -1       # an instance longer than the total
    assert lib.mrx_contours_write(*args, C.c_longlong(N.MRX_MAX_CONTOUR_SEGMENTS + 1),
                                  C.c_longlong(4), p16, p16, p16, p16, 1, 4, 8, None) == -2
    assert lib.mrx_contours_write(*args, C.c_longlong(10), C.c_longlong(4), None, p16, p16, p16,
                                  1, 4, 8, None) == -1       # no scratch for 10 segments
    assert N.contour_scratch_bytes(1000) == 48 * 1000 + 256


@pytest.mark.parametrize("S", [1, 4, 4095, 4096, 4097, 10 ** 6, 1 << 30])
def test_scratch_bound_holds_the_layout(S):
    """MRX_CONTOUR_SCRATCH_BYTES covers the layout contours.cu carves: 44 B per segment, aligned
    to 16, then one 8-byte sum per 4096-segment tile plus the total."""
    tiles = (S + 4095) // 4096
    need = ((44 * S + 15) & ~15) + 8 * (tiles + 1)
    assert need <= N.contour_scratch_bytes(S)
