"""CPU tests of Boundary IoU evaluation: the argument checks of mrx_mask_boundary and
mrx_coco_boundary_ious (every refused call returns before anything reaches the GPU), the
dilation_ratio checks of evaluate.COCOevalBoundary, and the host dilation table against the
restated mask_to_boundary (tests/boundary_cocoeval_oracle.py)."""
import ctypes as C

import numpy as np
import pytest

import boundary_cocoeval_oracle as bo
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N, evaluate
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import boundary_dilation

P = C.c_void_p(16)


def _refused(rc, fn, what):
    assert rc == -1, what
    assert N.load().mrx_last_error().decode().startswith(fn + ":"), what


def _boundary_args(null=None, B=1, R=100, max_w=64):
    p = [P] * 7
    if null is not None:
        p[null] = None
    return (*p, B, R, max_w, None)


@pytest.mark.parametrize("what,kw", [
    *[(f"null pointer {i}", dict(null=i)) for i in range(7)],
    ("null boundary with B = 0", dict(null=6, B=0)),
    ("B > MRX_MAX_BATCH", dict(B=N.MRX_MAX_BATCH + 1)),
    ("B < 0", dict(B=-1)),
    ("R = 0", dict(R=0)),
    ("R = 65535", dict(R=65535)),
    ("max_w = 0", dict(max_w=0)),
    ("negative max_w", dict(max_w=-8)),
])
def test_mask_boundary_refuses_bad_arguments(what, kw):
    _refused(N.load().mrx_mask_boundary(*_boundary_args(**kw)), "mrx_mask_boundary", what)


def test_mask_boundary_names_the_missing_regions():
    N.load().mrx_mask_boundary(*_boundary_args(null=4))
    assert "d_regions is required" in N.load().mrx_last_error().decode()


def _ious_args(null=None, B=1, R1=100, R2=100, packed1=P, boundary1=P):
    p = [P] * 19
    p[0], p[5] = packed1, boundary1
    if null is not None:
        p[null] = None
    return (*p[:9], R1, *p[9:18], R2, p[18], P, B, None)


@pytest.mark.parametrize("what,kw", [
    *[(f"null pointer {i}", dict(null=i)) for i in range(19)],
    ("null geometry with B = 0", dict(null=18, B=0)),
    ("B > MRX_MAX_BATCH", dict(B=N.MRX_MAX_BATCH + 1)),
    ("B < 0", dict(B=-1)),
    ("R1 = 0", dict(R1=0)),
    ("R1 = 65535", dict(R1=65535)),
    ("R2 = 0", dict(R2=0)),
    ("R2 = 65535", dict(R2=65535)),
    ("misaligned packed base", dict(packed1=C.c_void_p(17))),
    ("misaligned boundary base", dict(boundary1=C.c_void_p(18))),
])
def test_boundary_ious_refuse_bad_arguments(what, kw):
    _refused(N.load().mrx_coco_boundary_ious(*_ious_args(**kw)), "mrx_coco_boundary_ious", what)


def test_boundary_ious_null_iou_output():
    args = list(_ious_args())
    args[21] = None                                        # d_iou
    _refused(N.load().mrx_coco_boundary_ious(*args), "mrx_coco_boundary_ious", "null d_iou")


def test_empty_batches_launch_nothing():
    lib = N.load()
    assert lib.mrx_mask_boundary(*_boundary_args(B=0)) == 0
    assert lib.mrx_coco_boundary_ious(*_ious_args(B=0)) == 0


# ----------------------------------------------------------------------------- host side
@pytest.mark.parametrize("ratio", [0, -0.02, float("nan"), float("inf"), -float("inf"), "0.02",
                                   None, True, [0.02]])
def test_dilation_ratio_refusals(ratio):
    with pytest.raises(ValueError, match="dilation_ratio must be a finite number > 0"):
        evaluate.COCOevalBoundary(dilation_ratio=ratio)
    with pytest.raises(ValueError, match="dilation_ratio"):
        boundary_dilation([[4, 4, 4, 4, 0, 0, 4, 4]], ratio)


def test_dilation_ratio_is_frozen_after_the_first_batch():
    ev = evaluate.COCOevalBoundary(dilation_ratio=np.float32(0.25))
    assert ev.params.iouType == "boundary" and isinstance(ev.params.dilation_ratio, float)
    ev.add_batch([], [], [])                 # an empty batch freezes the parameters too
    ev.params.dilation_ratio = 0.03
    with pytest.raises(ValueError, match="dilation_ratio changed after the first batch"):
        ev.add_results([], [], [])
    ev.params.dilation_ratio = 0.25
    ev.add_results([], [], [])
    ev.accumulate()
    assert ev.eval["precision"].shape == (10, 101, 0, 4, 3)


def test_is_segm_with_the_iou_step_replaced():
    ev = evaluate.COCOevalBoundary(max_dets=(1, 5, 20), polygons=True, dilation_ratio=1)
    assert isinstance(ev, evaluate.COCOevalSegm) and ev._needs_masks and ev._polygons
    assert ev.params.maxDets == [1, 5, 20] and ev.params.dilation_ratio == 1.0
    for name in ("add_batch", "add_results", "evaluate", "accumulate", "summarize"):
        assert callable(getattr(ev, name))
    with pytest.raises(ValueError, match="polygon segmentations are not supported"):
        evaluate.COCOevalBoundary().add_results([], [[{"category_id": 1, "segmentation": [[0, 0, 1, 1, 2, 0]]}]], [1])


@pytest.mark.parametrize("ratio", [0.005, 0.02, 0.1, 0.5, 3.0, 1e12])
def test_host_dilation_table_equals_oracle(ratio):
    rng = np.random.default_rng(int(ratio * 1000) % 97)
    shapes = [(1024, 1024), (640, 480), (800, 1333), (2160, 3840), (5, 5), (1, 1), (37, 5)]
    shapes += [tuple(int(v) for v in rng.integers(1, 5000, size=2)) for _ in range(40)]
    geoms = [[h, w, h, w, 0, 0, h, w] for h, w in shapes]
    got = boundary_dilation(geoms, ratio)
    assert got.dtype == np.int32
    assert got.tolist() == [min(bo.dilation_of(h, w, ratio), 1 << 30) for h, w in shapes]


def test_round_half_to_even():
    # 0.5 * sqrt(3^2 + 4^2) = 2.5 rounds to 2; 0.5 * sqrt(6^2 + 8^2) = 5 stays 5
    assert boundary_dilation([[3, 4, 3, 4, 0, 0, 3, 4], [6, 8, 6, 8, 0, 0, 6, 8]], 0.5).tolist() \
        == [bo.dilation_of(3, 4, 0.5), bo.dilation_of(6, 8, 0.5)] == [2, 5]
    assert boundary_dilation([[3, 4, 3, 4, 0, 0, 3, 4]], 0.7).tolist() == [bo.dilation_of(3, 4, 0.7)]
