"""Detection rows the model does not normally produce, against NumPy's reading of them.

Steps 1-6 of upstream `unmold_detections` trim the list at the first class_id == 0, cast class
ids with astype(int32) (truncation; NaN and out-of-range values become INT_MIN on x86), gather
mrcnn_mask[..., class_ids] (negative ids index from the end, anything outside [-C, C) raises
IndexError, before zero-area rows are dropped), and paste each mask with
full_mask[y1:y2, x1:x2] = mask (a box partly outside the image raises ValueError).

Every case runs through UnmoldEngine with the tile buffer filled with 1.0 first, so that a tile
the class gather never wrote would expand to a full box instead of passing by luck."""
import numpy as np
import pytest

import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import synth
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import UnmoldEngine, make_geom

from helpers import canvas_masks, compare_masks, oracle_unmold

pytestmark = pytest.mark.gpu

H, W = 48, 64
R = 8
C = 5
ROW = 2              # the row each case changes
BOXES = [(2, 3, 20, 30), (10, 10, 40, 60), (0, 0, H, W), (30, 5, 47, 25), (5, 40, 12, 63),
         (1, 1, 9, 9)]


def _image(class_id=None, box=None, classes=C, all_class_ids=None):
    """Six detections with exact pixel boxes on an unscaled mold (molded == original pixels);
    row ROW gets `class_id` / `box` when given."""
    rng = np.random.default_rng(31)
    im = synth.make_image(rng, (H, W), len(BOXES), num_classes=max(classes, 2), max_instances=R,
                          mold=((H, W, 3), (0, 0, H, W)))
    im.mrcnn_mask = np.ascontiguousarray(im.mrcnn_mask[..., :classes])
    boxes = list(BOXES)
    if box is not None:
        boxes[ROW] = box
    im.detections[:len(boxes), :4] = synth._norm_boxes_f32(np.array(boxes, np.float64), (H, W))
    if all_class_ids is not None:
        im.detections[:len(boxes), 4] = all_class_ids
    if class_id is not None:
        im.detections[ROW, 4] = class_id
    return im


def _device(im, dtype):
    import torch

    classes = im.mrcnn_mask.shape[-1]
    eng = UnmoldEngine(1, R, (28, 28), classes, det_dtype=dtype, mask_dtype=dtype)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window)])
    eng.d_tiles.fill_(1.0)
    d_det = torch.from_numpy(im.detections.astype(dtype)[None]).cuda()
    d_msk = torch.from_numpy(im.mrcnn_mask.astype(dtype)[None]).cuda()
    eng.enqueue(d_det, d_msk)
    counts, boxes, cls, scores = eng.fetch_meta()
    k = int(counts[0])
    return boxes[0, :k].copy(), cls[0, :k].copy(), scores[0, :k].copy(), canvas_masks(eng, 0, k)


def _reference(im, dtype):
    with np.errstate(invalid="ignore"):      # NaN -> int32 warns, then indexes with INT_MIN
        return oracle_unmold(im, dtype, return_resized=True)


def _same_as_numpy(im, dtype):
    """The device result equals the oracle's, or both raise the same exception type.  Returns
    the oracle result (None when it raised)."""
    try:
        rb, rc, rs, rm, rz = _reference(im, dtype)
    except (IndexError, ValueError) as e:
        with pytest.raises(type(e)):
            _device(im, dtype)
        return None
    b, c, s, m = _device(im, dtype)
    np.testing.assert_array_equal(b, rb)
    np.testing.assert_array_equal(c, rc)
    np.testing.assert_array_equal(s, rs)
    assert m.shape == rm.shape
    assert compare_masks(m, rm, rz, rb)[0] == 0
    return rb, rc, rs, rm


DTYPES = pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])


@DTYPES
@pytest.mark.parametrize("class_id", [0.5, -0.5, 0.999])
def test_class_id_truncating_to_zero_keeps_the_row(cuda_device, dtype, class_id):
    """Not 0, so it does not end the list; astype(int32) makes it class 0, whose tile is used."""
    rb, rc, rs, rm = _same_as_numpy(_image(class_id), dtype)
    assert len(rb) == len(BOXES) and rc[ROW] == 0


@DTYPES
def test_negative_zero_class_id_ends_the_list(cuda_device, dtype):
    rb, rc, rs, rm = _same_as_numpy(_image(-0.0), dtype)
    assert len(rb) == ROW


@DTYPES
@pytest.mark.parametrize("class_id", [-1.0, float(-C)])
def test_negative_class_id_indexes_from_the_end(cuda_device, dtype, class_id):
    rb, rc, rs, rm = _same_as_numpy(_image(class_id), dtype)
    assert len(rb) == len(BOXES) and rc[ROW] == int(class_id)


@DTYPES
@pytest.mark.parametrize("class_id", [float("nan"), float(C), float(-C - 1), 3e9])
def test_class_id_numpy_cannot_index_raises(cuda_device, dtype, class_id):
    with pytest.raises(IndexError):
        _reference(_image(class_id), dtype)
    assert _same_as_numpy(_image(class_id), dtype) is None


@DTYPES
def test_class_id_out_of_range_on_a_zero_area_row_raises(cuda_device, dtype):
    """NumPy gathers the class tiles before it drops zero-area rows."""
    im = _image(float(C + 2), box=(5, 20, 30, 20))
    with pytest.raises(IndexError):
        _reference(im, dtype)
    assert _same_as_numpy(im, dtype) is None


@DTYPES
def test_single_class_with_class_id_minus_one(cuda_device, dtype):
    rb, rc, rs, rm = _same_as_numpy(_image(classes=1, all_class_ids=-1.0), dtype)
    assert len(rb) == len(BOXES) and (rc == -1).all()


@DTYPES
@pytest.mark.parametrize("box", [(30, 5, H + 2, 25), (5, -3, 20, 25), (-2, 5, 20, 25),
                                 (5, 40, 20, W + 6)],
                         ids=["y2_below", "x1_left", "y1_above", "x2_right"])
def test_box_partly_outside_the_image_raises(cuda_device, dtype, box):
    with pytest.raises(ValueError):
        _reference(_image(box=box), dtype)
    assert _same_as_numpy(_image(box=box), dtype) is None


@DTYPES
def test_inverted_box_with_positive_area_raises(cuda_device, dtype):
    """(y2 - y1) * (x2 - x1) > 0 with both extents negative: the row is kept, and neither the
    reference's resize (negative dimensions) nor the device can paste it."""
    im = _image(box=(20, 30, 5, 10))
    with pytest.raises(ValueError):
        _reference(im, dtype)
    assert _same_as_numpy(im, dtype) is None


@DTYPES
def test_box_entirely_at_negative_rows_raises_where_numpy_wraps(cuda_device, dtype):
    """NumPy slicing wraps negative indices, so the reference pastes a box that lies entirely at
    negative rows into the last rows of the image.  The device does not reproduce the wrap; it
    raises ValueError, as for any box outside the image."""
    box = (-6, 2, -1, 9)
    im = _image(box=box)
    rb, rc, rs, rm, rz = _reference(im, dtype)
    assert tuple(rb[ROW]) == box
    plane = rm[:, :, ROW]
    want = np.zeros((H, W), bool)
    want[H - 6:H - 1, 2:9] = rz[ROW] >= 0.5
    assert np.array_equal(plane, want) and want.any()
    with pytest.raises(ValueError):
        _device(im, dtype)
