"""The expand kernels over the mask-tile shapes the C ABI accepts (2 <= mh <= 64, 4 <= mw <= 64,
mw % 4 == 0; square or not), not only the 28x28 tiles of the model.

Tiles up to MRX_MAX_LANE_MASK_W (30) columns wide take the team kernel, whose fast and general paths, six-row queue and
lane-column clamps all depend on mh and mw; the bit-packed and RLE kernels compute the same
sample.  Wider tiles take the generic kernel, which stages two tile rows per canvas row.  Every
shape runs boxes of every size relative to the tile: 1 px, smaller than the tile (downscale),
a few tiles, and the whole canvas."""
import numpy as np
import pytest

import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, synth

from helpers import (canvas_masks, check_values, compare_masks, item_of, oracle_unmold,
                     prepared_engine)

pytestmark = pytest.mark.gpu

HW = (240, 333)          # an odd width: canvas rows are not 16-byte aligned
R = 48
CLASSES = 3

TEAM_SHAPES = [(2, 4), (3, 8), (5, 12), (7, 28), (14, 16), (28, 4), (28, 20), (33, 24), (56, 28),
               (64, 8), (64, 28)]
GENERIC_SHAPES = [(2, 64), (13, 44), (28, 60), (56, 56), (64, 36), (64, 64)]


def _images(mask_hw, seed):
    """Two images: one molded the usual way with boxes from 1 px to the whole window, and one
    unscaled (molded == original pixels) with tiny boxes, an exact 1x1 box, a whole-canvas box
    and a zero-area row (kept instance k then resizes tile k + 1)."""
    rng = np.random.default_rng(seed)
    H, W = HW
    a = synth.make_image(rng, HW, 40, num_classes=CLASSES, max_instances=R, mask_hw=mask_hw,
                         min_box=1, max_box_frac=1.0)
    b = synth.make_image(rng, HW, 36, num_classes=CLASSES, max_instances=R, mask_hw=mask_hw,
                         min_box=1, max_box_frac=0.05, zero_area_rows=(3,),
                         mold=((H, W, 3), (0, 0, H, W)))
    exact = np.array([[17, 40, 18, 41], [0, 0, H, W]], np.float64)
    b.detections[:2, :4] = synth._norm_boxes_f32(exact, (H, W))
    return [a, b]


def _expanded(ims, mask_hw):
    eng = prepared_engine(ims, R, CLASSES, np.float64, mask_hw)
    eng.enqueue_expand()
    counts, boxes, cls, scores = eng.fetch_meta()
    return eng, [int(c) for c in counts], boxes, cls, scores


def _check_pack_masks(eng, ims, counts):
    """mrx_pack_masks over the byte canvas equals np.packbits of it, plane for plane."""
    eng._packed_buffer()
    eng.d_packed.fill_(0xAA)       # poison: every packed byte must be rewritten
    d_packed, off = eng.pack_masks()
    _check_packed(eng, ims, counts, d_packed, off)


def _check_packed(eng, ims, counts, d_packed, off):
    for b, (im, k) in enumerate(zip(ims, counts)):
        H, W = im.original_image_shape[:2]
        wb = (W + 7) // 8
        got = d_packed[int(off[b]):int(off[b]) + k * H * wb].cpu().numpy().reshape(k, H, wb)
        want = np.packbits(canvas_masks(eng, b, k).transpose(2, 0, 1), axis=-1)
        assert np.array_equal(got, want), f"image {b}"


def _check_rle(eng, ims, counts):
    """mrx_rle_* equals the oracle's RLE of the byte canvas, instance for instance."""
    d_runs, off = eng.enqueue_rle()
    runs = d_runs.cpu().numpy().view(np.uint32)
    for b, (im, k) in enumerate(zip(ims, counts)):
        m = canvas_masks(eng, b, k)
        for n in range(k):
            i = b * eng.R + n
            want = oracle.rle_encode(m[:, :, n])["counts"]
            assert np.array_equal(runs[int(off[i]) + i:int(off[i + 1]) + i + 1], want), (b, n)


@pytest.mark.parametrize("mask_hw", TEAM_SHAPES, ids=[f"{h}x{w}" for h, w in TEAM_SHAPES])
def test_team_kernel_tile_shape(cuda_device, mask_hw):
    ims = _images(mask_hw, 500 + mask_hw[0] * 64 + mask_hw[1])
    # values within 1e-6 of float64, masks equal outside the band, plain launch == values launch
    check_values(f"tile_shape/{mask_hw[0]}x{mask_hw[1]}", ims, R, CLASSES, mask_hw=mask_hw)
    eng, counts, _, _, _ = _expanded(ims, mask_hw)
    d_packed, off = eng.enqueue_expand_packed()
    _check_packed(eng, ims, counts, d_packed, off)
    _check_rle(eng, ims, counts)
    _check_pack_masks(eng, ims, counts)


@pytest.mark.parametrize("mask_hw", GENERIC_SHAPES, ids=[f"{h}x{w}" for h, w in GENERIC_SHAPES])
def test_generic_kernel_tile_shape(cuda_device, mask_hw):
    import torch

    ims = _images(mask_hw, 600 + mask_hw[0] * 64 + mask_hw[1])
    eng, counts, boxes, cls, scores = _expanded(ims, mask_hw)
    for b, im in enumerate(ims):
        rb, rc, rs, rm, rz = oracle_unmold(im, np.float64, return_resized=True)
        k = counts[b]
        np.testing.assert_array_equal(boxes[b, :k], rb)
        np.testing.assert_array_equal(cls[b, :k], rc)
        np.testing.assert_array_equal(scores[b, :k], rs)
        assert compare_masks(canvas_masks(eng, b, k), rm, rz, rb)[0] == 0
    _check_pack_masks(eng, ims, counts)
    # the kernels that need a tile row in one warp's lanes refuse the shape before launching
    with pytest.raises(N.MrxError, match=r"status -2"):
        eng.enqueue_expand_packed()
    with pytest.raises(N.MrxError, match=r"status -2"):
        eng.enqueue_rle()
    with pytest.raises(N.MrxError, match=r"status -2"):
        eng.enqueue_expand_values(torch.empty(int(eng._offsets[2]), dtype=torch.float32,
                                              device="cuda"))
    with pytest.raises(N.MrxError, match=r"status -2"):
        api_utils.unmold_detections_rle_batch([item_of(im) for im in ims])


@pytest.mark.parametrize("mask_hw", [(1, 28), (28, 6)], ids=["mh1", "mw6"])
def test_tile_shape_no_kernel_takes_raises(cuda_device, mask_hw):
    """mrx_unmold_prepare gathers tiles of any shape, but no expand kernel takes these: every
    call must fail rather than return masks."""
    rng = np.random.default_rng(7)
    im = synth.make_image(rng, (64, 80), 5, num_classes=CLASSES, max_instances=8, mask_hw=mask_hw)
    with pytest.raises(N.MrxError, match=r"mrx_mask_expand failed \(status -2\)"):
        api_utils.unmold_detections(*item_of(im))
    with pytest.raises(N.MrxError, match=r"mrx_mask_expand_packed failed \(status -2\)"):
        api_utils.unmold_detections_packed_batch([item_of(im)])
    with pytest.raises(N.MrxError, match=r"mrx_rle_count failed \(status -2\)"):
        api_utils.unmold_detections_rle_batch([item_of(im)])
