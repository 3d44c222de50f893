"""Mask contour polygons traced on the device (extension of display_instances' polygon loop):
every polygon must equal, exactly and in the same order, the restated
`np.fliplr(find_contours(padded_mask, 0.5)) - 1` of the mask `unmold_detections` returns."""
import numpy as np
import pytest

import contour_oracle as co
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, synth, visualize

from helpers import item_of, prepared_engine

pytestmark = pytest.mark.gpu


def _assert_same(got, want, what=""):
    assert len(got) == len(want), (what, len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w), (what, i, len(g), len(w))
        for j, (a, b) in enumerate(zip(g, w)):
            assert a.dtype == np.float64 and a.shape == b.shape, (what, i, j, a.shape, b.shape)
            assert np.array_equal(a, b), (what, i, j)


def _check(ims, dtype=np.float32):
    items = [item_of(im, dtype) for im in ims]
    got = api_utils.unmold_detections_contours_batch(items)
    ref = api_utils.unmold_detections_batch(items)
    verts = 0
    for b, ((bx, c, s, polys), (rb, rc, rs, rm)) in enumerate(zip(got, ref)):
        assert np.array_equal(bx, rb) and np.array_equal(c, rc) and np.array_equal(s, rs)
        _assert_same(polys, co.mask_polygons(rb, rm), f"image {b}")
        verts += sum(len(v) for p in polys for v in p)
    return verts


@pytest.mark.parametrize("hw,n,R,kw", [
    ((96, 128), 12, 16, {}),
    ((64, 96), 40, 40, dict(min_box=60, max_box_frac=1.0)),     # full-height / full-width boxes
    ((40, 56), 30, 32, dict(min_box=20, max_box_frac=1.0)),     # boxes touching every border
    ((150, 150), 30, 32, dict(min_box=1, max_box_frac=0.1)),    # boxes smaller than the tile
    ((75, 333), 37, 40, {}),                                    # widths no multiple of 8 / 32
    ((33, 1000), 7, 8, {}),
    ((17, 9), 3, 4, dict(min_box=1, max_box_frac=1.0)),
    ((64, 80), 0, 4, {}),                                       # nothing detected
])
def test_contours_equal_oracle(cuda_device, hw, n, R, kw):
    rng = np.random.default_rng(91)
    ims = [synth.make_image(rng, hw, n, num_classes=4, max_instances=R, **kw) for _ in range(3)]
    _check(ims)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_contours_full_size(cuda_device, dtype):
    """configs[1] images (100 and 37 instances) and an 800x1333 batch with zero-area drops."""
    ims = synth.make_batch(93, 1, (1024, 1024), 100) + synth.make_batch(94, 1, (1024, 1024), 37)
    assert _check(ims, dtype) > 0
    rng = np.random.default_rng(95)
    ims = [synth.make_image(rng, (800, 1333), 60, num_classes=81, max_instances=100,
                            zero_area_rows=(2, 30, 59)) for _ in range(2)]
    _check(ims, dtype)


def test_contours_mixed_shapes_and_an_empty_image(cuda_device):
    rng = np.random.default_rng(96)
    ims = [synth.make_image(rng, hw, n, num_classes=5, max_instances=24, mold=mold)
           for hw, n, mold in [((120, 200), 20, None), ((64, 64), 0, None), ((333, 75), 24, None),
                               ((90, 90), 7, ((128, 128, 3), (19, 19, 109, 109)))]]
    _check(ims)


def test_contours_wide_tiles_take_the_canvas_route(cuda_device):
    rng = np.random.default_rng(97)
    ims = [synth.make_image(rng, (140, 171), 20, num_classes=4, max_instances=24, mask_hw=(24, 32))
           for _ in range(2)]
    _check(ims)


def test_packed_routes_give_identical_contours(cuda_device):
    """The planes of mrx_mask_expand_packed and of mrx_mask_expand + mrx_pack_masks trace to the
    same polygons; and a second batch on the same engine reuses its buffers correctly."""
    rng = np.random.default_rng(98)
    a = [synth.make_image(rng, (300, 411), 50, num_classes=6, max_instances=64) for _ in range(3)]
    b = [synth.make_image(rng, (300, 411), 64, num_classes=6, max_instances=64, min_box=40,
                          max_box_frac=1.0) for _ in range(3)]
    eng = prepared_engine(a, 64, 6, np.float32)
    eng.enqueue_expand_packed()
    direct = eng.enqueue_contours()
    eng.enqueue_expand()
    eng.pack_masks()
    via_canvas = eng.enqueue_contours()
    for b_, (p, q) in enumerate(zip(direct, via_canvas)):
        _assert_same(p, q, f"image {b_}")
    ref = api_utils.unmold_detections_batch([item_of(im, np.float32) for im in a])
    for (rb, _, _, rm), p in zip(ref, direct):
        _assert_same(p, co.mask_polygons(rb, rm))
    # second batch, more segments, on the same engine
    import torch

    eng.plan([eng._geom_host[0]] * 3)
    d_det = torch.from_numpy(np.stack([im.detections.astype(np.float32) for im in b])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask.astype(np.float32) for im in b])).cuda()
    eng.enqueue_packed(d_det, d_msk)
    second = eng.enqueue_contours()
    ref = api_utils.unmold_detections_batch([item_of(im, np.float32) for im in b])
    for (rb, _, _, rm), p in zip(ref, second):
        _assert_same(p, co.mask_polygons(rb, rm))


def _masks_cases():
    rng = np.random.default_rng(99)
    single = np.zeros((5, 6), bool)
    single[2, 3] = True
    diag = np.zeros((4, 4), bool)
    diag[1, 1] = diag[2, 2] = True
    checker = (np.indices((8, 8)).sum(0) % 2).astype(bool)    # both saddle cases
    ring = np.zeros((7, 7), bool)
    ring[1:6, 1:6] = True
    ring[2:5, 2:5] = False
    island = np.zeros((9, 9), bool)                           # a blob inside a hole
    island[1:8, 1:8] = True
    island[2:7, 2:7] = False
    island[4, 4] = True
    return [
        ("single_pixel", single), ("diagonal", diag), ("checkerboard", checker), ("ring", ring),
        ("blob_in_hole", island), ("all_ones", np.ones((6, 9), bool)),
        ("empty", np.zeros((5, 5), bool)), ("1x1", np.ones((1, 1), bool)),
        ("1xW", rng.random((1, 37)) < 0.5), ("Hx1", rng.random((29, 1)) < 0.5),
        ("noise_64x1333", rng.random((64, 1333)) < 0.5),
    ]


@pytest.mark.parametrize("name,mask", _masks_cases())
def test_mask_contours_numpy_entry(cuda_device, name, mask):
    H, W = mask.shape
    masks = np.stack([mask, ~mask, mask], axis=-1)
    boxes = np.array([[0, 0, H, W], [0, 0, H, W], [0, 0, 0, 0]], np.int32)   # the last is skipped
    got = visualize.mask_contours(boxes, masks)
    assert got[2] == []
    _assert_same(got, co.mask_polygons(boxes, masks), name)
