"""CPU tests of COCO box evaluation: the argument checks of mrx_coco_box_ious and
mrx_coco_match_f64area (every refused call returns before anything reaches the GPU), the
ValueErrors of evaluate.COCOevalBbox, and known answers of the restated bbIou
(tests/bbox_cocoeval_oracle.py)."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

import bbox_cocoeval_oracle as bo
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N, evaluate

P = C.c_void_p(16)


def _refused(rc, fn, what):
    assert rc == -1, what
    assert N.load().mrx_last_error().decode().startswith(fn + ":"), what


def _box_ious_args(null=None, B=1, R1=100, R2=100, form=N.MRX_BOX_YXYX_I32):
    p = [P] * 10
    if null is not None:
        p[null] = None
    return (p[0], form, p[1], p[2], p[3], R1, p[4], p[5], p[6], p[7], R2, p[8], p[9], B, None)


@pytest.mark.parametrize("what,kw", [
    *[(f"null pointer {i}", dict(null=i)) for i in range(10)],
    ("null pointer with B = 0", dict(null=9, B=0)),
    ("B > MRX_MAX_BATCH", dict(B=N.MRX_MAX_BATCH + 1)),
    ("B < 0", dict(B=-1)),
    ("R1 = 0", dict(R1=0)),
    ("R1 = 65535", dict(R1=65535)),
    ("R2 = 0", dict(R2=0)),
    ("R2 = 65535", dict(R2=65535)),
    ("bad box form", dict(form=2)),
    ("negative box form", dict(form=-1)),
])
def test_box_ious_refuses_bad_arguments(what, kw):
    _refused(N.load().mrx_coco_box_ious(*_box_ious_args(**kw)), "mrx_coco_box_ious", what)


def _match_args(null=None, B=1, R1=100, R2=100, T=10, A=4):
    p = [P] * 12
    thr = N.double_array([0.5] * max(T, 1))
    rng = N.double_array([0.0, 1e10] * max(A, 1))
    args = [*p[:10], thr, T, rng, A, p[10], p[11], B, R1, R2, None]
    if null is not None:
        args[[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 15][null]] = None
    return args


@pytest.mark.parametrize("what,kw", [
    *[(f"null pointer {i}", dict(null=i)) for i in range(14)],
    ("null thresholds with B = 0", dict(null=10, B=0)),
    ("B > MRX_MAX_BATCH", dict(B=N.MRX_MAX_BATCH + 1)),
    ("B < 0", dict(B=-1)),
    ("R1 = 0", dict(R1=0)),
    ("R1 = 65535", dict(R1=65535)),
    ("R2 = 0", dict(R2=0)),
    ("R2 = 65535", dict(R2=65535)),
    ("T = 0", dict(T=0)),
    ("T above MRX_MAX_IOU_THRESHOLDS", dict(T=N.MRX_MAX_IOU_THRESHOLDS + 1)),
    ("A = 0", dict(A=0)),
    ("A above MRX_MAX_AREA_RANGES", dict(A=N.MRX_MAX_AREA_RANGES + 1)),
])
def test_match_f64area_refuses_bad_arguments(what, kw):
    _refused(N.load().mrx_coco_match_f64area(*_match_args(**kw)), "mrx_coco_match_f64area", what)


def test_empty_batches_launch_nothing():
    lib = N.load()
    for form in (N.MRX_BOX_YXYX_I32, N.MRX_BOX_XYWH_F64):
        assert lib.mrx_coco_box_ious(*_box_ious_args(B=0, form=form)) == 0
    assert lib.mrx_coco_match_f64area(*_match_args(B=0, T=N.MRX_MAX_IOU_THRESHOLDS,
                                                   A=N.MRX_MAX_AREA_RANGES)) == 0


# ----------------------------------------------------------------------------- host refusals
ITEM = (np.zeros((2, 6), np.float32), np.zeros((2, 28, 28, 3), np.float32), (4, 6, 3),
        (16, 16, 3), (0, 0, 11, 16))
GT = {"category_id": 1, "bbox": [0, 0, 2, 2], "area": 4.0, "id": 7}
RES = {"image_id": 1, "category_id": 1, "score": 0.5, "bbox": [0, 0, 2, 2]}


def _gt(**kw):
    g = dict(GT, **kw)
    return {k: v for k, v in g.items() if v is not None}


@pytest.mark.parametrize("ann,msg", [
    (_gt(bbox=None), r"image 1, annotation 0 \(id 7\): no 'bbox'"),
    (_gt(area=None), r"image 1, annotation 0 \(id 7\): no 'area'"),
    (_gt(bbox=[0, 0, 2]), "bbox must be 4 numbers"),
    (_gt(bbox=[0, 0, 2, 2, 2]), "bbox must be 4 numbers"),
    (_gt(bbox=[[0, 0], [2, 2]]), "bbox must be 4 numbers"),
    (_gt(bbox=["a", 0, 2, 2]), "bbox must be 4 numbers"),
    (_gt(bbox=[0, np.nan, 2, 2]), "not finite"),
    (_gt(bbox=[0, 0, np.inf, 2]), "not finite"),
    (_gt(bbox=[1.7e308, 0, 1.7e308, 2]), "not finite"),           # x + w overflows
    (_gt(bbox=[0, 0, 1e200, 1e200]), "not finite"),               # w * h overflows
    (_gt(area=float("nan")), "area is NaN"),
])
@pytest.mark.parametrize("via", ["add_batch", "add_results"])
def test_ground_truth_refusals(ann, msg, via):
    ev = evaluate.COCOevalBbox()
    with pytest.raises(ValueError, match=msg):
        if via == "add_batch":
            ev.add_batch([ITEM], [1], [[ann]])
        else:
            ev.add_results([], [[ann]], [1])


def test_segmentation_is_not_read():
    """A polygon, an RLE dict, garbage or no segmentation at all: the tables are built without
    touching it."""
    ev = evaluate.COCOevalBbox()
    anns = [_gt(segmentation=s) for s in ([[0, 0, 1, 1, 2, 0]], {"size": [9, 9], "counts": b"x"},
                                          "garbage", None)]
    cats, crowd, area, boxes = ev._gt_tables([1], [anns])
    assert boxes[0].shape == (4, 4) and area[0].tolist() == [4.0] * 4


@pytest.mark.parametrize("res,msg", [
    (dict(RES, image_id=9), "result 0: image 9 is not one"),
    ({k: v for k, v in RES.items() if k != "bbox"}, "result 0: no 'bbox'"),
    (dict(RES, bbox=[0, 0, 1]), "result 0: bbox must be 4 numbers"),
    (dict(RES, bbox=[0, 0, float("nan"), 1]), "result 0: bbox .* is not finite"),
    (dict(RES, bbox=[0, 0, 1e300, 1e300]), "result 0: bbox .* is not finite"),
])
def test_result_refusals(res, msg):
    with pytest.raises(ValueError, match=msg):
        evaluate.COCOevalBbox().add_results([res], [[GT]], [1])


def test_batch_checks():
    ev = evaluate.COCOevalBbox()
    with pytest.raises(ValueError, match="1 items but 2 image ids"):
        ev.add_batch([ITEM], [1, 2], [[], []])
    with pytest.raises(ValueError, match="image 3 was already added"):
        ev.add_batch([ITEM, ITEM], [3, 3], [[], []])
    ev._img_index[5] = 0
    with pytest.raises(ValueError, match="image 5 was already added"):
        ev.add_results([], [[]], [5])


def test_params_and_api():
    ev = evaluate.COCOevalBbox(max_dets=(1, 5, 20))
    assert ev.params.iouType == "bbox" and evaluate.COCOevalSegm().params.iouType == "segm"
    assert ev.params.maxDets == [1, 5, 20]
    for name in ("add_batch", "add_results", "evaluate", "accumulate", "summarize"):
        assert callable(getattr(ev, name))
    ev.add_batch([], [], [])          # an empty batch is fine and changes nothing
    ev.accumulate()
    assert ev.eval["precision"].shape == (10, 101, 0, 4, 3)


def test_the_same_evaluator_twice_is_refused():
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils

    ev = evaluate.COCOevalBbox()
    with pytest.raises(ValueError, match="given twice"):
        api_utils.unmold_coco_eval_batch([ITEM], [1], [[]], [ev, ev])


# ----------------------------------------------------------------------------- oracle answers
# boxes whose unfused u = (da + ga) - w*h and fused fma(-w, h, da + ga) round apart, so the IoUs
# differ (found with fractions.Fraction over random boxes with 2-decimal coordinates)
FUSED_D = [2.03, 406.76, 135.82, 124.67]
FUSED_G = [33.88, 404.83, 127.0, 193.01]


def fused_iou(D, G):
    """bbIou with da + ga - w*h contracted into one FMA (what nvcc does unless told not to)."""
    w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
    h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
    i = w * h
    u = float(Fraction(D[2] * D[3] + G[2] * G[3]) - Fraction(w) * Fraction(h))
    return i / u


def test_known_answers():
    a, b = [0, 0, 10, 10], [5, 5, 10, 10]
    assert bo.bb_iou([a], [b], [0])[0, 0] == 1 / 7
    assert bo.bb_iou([a], [b], [1])[0, 0] == 0.25
    assert bo.bb_iou([a], [[10, 0, 5, 5], [0, 10, 5, 5], [-5, -5, 5, 5]], None).tolist() == \
        [[0.0, 0.0, 0.0]]                         # touching boxes
    assert bo.bb_iou([[0, 0, -3, 10], [0, 0, 0, 10]], [a], [0]).tolist() == [[0.0], [0.0]]
    assert bo.bb_iou([a], [a], [0])[0, 0] == 1.0
    assert bo.bb_iou([], [a], [0]).shape == (0, 1)


def test_fused_pair_rounds_apart():
    got = bo.bb_iou([FUSED_D], [FUSED_G], [0])[0, 0]
    D, G = FUSED_D, FUSED_G
    w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
    h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
    assert got == (w * h) / (D[2] * D[3] + G[2] * G[3] - w * h)
    assert got != fused_iou(D, G)


def test_oracle_detection_area_is_loadres():
    ev = bo.COCOevalBboxOracle(
        [{"image_id": 1, "category_id": 1, "bbox": [0, 0, 4, 4], "iscrowd": 0, "area": 16.0}],
        [{"image_id": 1, "category_id": 1, "bbox": [0.5, 0, 2.5, 1.5], "score": 0.5}])
    ev.evaluate()
    assert ev._dts[1, 1][0]["area"] == 3.75
    assert ev.ious[1, 1][0, 0] == 3.75 / 16
