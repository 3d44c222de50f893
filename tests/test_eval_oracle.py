"""CPU tests of the mask-scoring restatement (tests/eval_oracle.py) on answers worked by hand, of
the closed form of its matching loop that mrx_mask_matches computes, and of the host helpers of
`evaluate` (threshold conversion, AP tail) against it."""
import numpy as np
import pytest

import eval_oracle as eo
from matterport_maskrcnn_with_tensorflow_serving_b200 import evaluate
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import comparison_threshold


def _square(H, W, y1, x1, y2, x2):
    m = np.zeros((H, W), bool)
    m[y1:y2, x1:x2] = True
    return m


def _case(gt, pred, gt_cls=None, pred_cls=None, scores=None):
    """(gt_boxes, gt_class_ids, gt_masks, pred_boxes, pred_class_ids, pred_scores, pred_masks)
    from lists of [H, W] masks; boxes are all ones (never trimmed) unless given."""
    gm = np.stack(gt, -1) if gt else np.zeros((8, 8, 0), bool)
    pm = np.stack(pred, -1) if pred else np.zeros((8, 8, 0), bool)
    n, m = pm.shape[-1], gm.shape[-1]
    return (np.ones((m, 4), np.int32), np.asarray(gt_cls if gt_cls is not None else [1] * m),
            gm, np.ones((n, 4), np.int32), np.asarray(pred_cls if pred_cls is not None else [1] * n),
            np.asarray(scores if scores is not None else np.linspace(0.9, 0.5, n), np.float32), pm)


def test_iou_of_squares_sharing_one_pixel():
    a = _square(4, 4, 0, 0, 2, 2)[..., None]
    b = _square(4, 4, 1, 1, 3, 3)[..., None]
    ov = eo.compute_overlaps_masks(a, b)
    assert ov.dtype == np.float32 and ov[0, 0] == np.float32(1 / 7)


def test_ap_of_one_miss_between_two_hits():
    g0, g1 = _square(16, 16, 0, 0, 4, 4), _square(16, 16, 8, 8, 12, 12)
    miss = _square(16, 16, 0, 10, 3, 14)
    args = _case([g0, g1], [g0, miss, g1], scores=[0.9, 0.8, 0.7])
    ap, precisions, recalls, _ = eo.compute_ap(*args)
    gt_match, pred_match, _ = eo.compute_matches(*args)
    assert pred_match.tolist() == [0, -1, 1] and gt_match.tolist() == [0, 2]
    assert ap == 0.8333333333333333 and ap.dtype == np.float64
    got = evaluate.ap_from_matches(pred_match, gt_match)
    assert got[0] == ap and np.array_equal(got[1], precisions) and np.array_equal(got[2], recalls)


def test_class_mismatch_is_skipped():
    g = _square(16, 16, 0, 0, 10, 10)
    near = _square(16, 16, 0, 0, 10, 9)                       # IoU 0.9, other class
    far = _square(16, 16, 0, 0, 10, 6)                        # IoU 0.6, same class
    args = _case([near, far], [g], gt_cls=[2, 1], pred_cls=[1])
    assert eo.compute_matches(*args)[1].tolist() == [1]
    args = _case([near, far], [g], gt_cls=[2, 3], pred_cls=[1])
    assert eo.compute_matches(*args)[1].tolist() == [-1]


def test_matched_gt_is_skipped():
    g0, g1 = _square(16, 16, 0, 0, 10, 10), _square(16, 16, 0, 0, 10, 8)
    args = _case([g0, g1], [g0, g0])
    gt_match, pred_match, _ = eo.compute_matches(*args)
    assert pred_match.tolist() == [0, 1] and gt_match.tolist() == [0, 1]


def test_tie_takes_the_larger_gt_index():
    g = _square(16, 16, 2, 2, 9, 9)
    gt_match, pred_match, _ = eo.compute_matches(*_case([g, g, g], [g]))
    assert pred_match.tolist() == [2] and gt_match.tolist() == [-1, -1, 0]


def test_equal_scores_rank_the_larger_index_first():
    g0, g1 = _square(16, 16, 0, 0, 4, 4), _square(16, 16, 8, 8, 12, 12)
    gt_match, pred_match, ov = eo.compute_matches(*_case([g0, g1], [g0, g1], scores=[0.5, 0.5]))
    assert pred_match.tolist() == [1, 0] and ov[0, 1] == 1 and ov[1, 0] == 1


def test_empty_prediction_matches_empty_gt_by_nan():
    e = np.zeros((8, 8), bool)
    gt_match, pred_match, ov = eo.compute_matches(*_case([e], [e]))
    assert np.isnan(ov[0, 0]) and pred_match.tolist() == [0]


def test_score_threshold_cuts_candidates():
    g, p = _square(16, 16, 0, 0, 10, 10), _square(16, 16, 0, 0, 10, 6)   # IoU 0.6
    args = _case([g], [p])
    assert eo.compute_matches(*args, iou_threshold=0.5)[1].tolist() == [0]
    assert eo.compute_matches(*args, iou_threshold=0.5, score_threshold=0.7)[1].tolist() == [-1]


def test_float32_against_float64_threshold():
    """IoU 7000/10000 rounds to float32(0.7): a Python 0.7 compares in float32 (equal, a match),
    np.float64(0.7) in float64 (float32(0.7) < 0.7, no match)."""
    g, p = _square(100, 100, 0, 0, 100, 100), _square(100, 100, 0, 0, 70, 100)
    args = _case([g], [p])
    assert eo.compute_overlaps_masks(p[..., None], g[..., None])[0, 0] == np.float32(0.7)
    assert eo.compute_matches(*args, iou_threshold=0.7)[1].tolist() == [0]
    assert eo.compute_matches(*args, iou_threshold=np.float64(0.7))[1].tolist() == [-1]
    assert comparison_threshold(0.7) == float(np.float32(0.7))
    assert comparison_threshold(np.float64(0.7)) == 0.7


def test_no_gt_and_no_predictions():
    g = _square(16, 16, 0, 0, 4, 4)
    ap, _, _, ov = eo.compute_ap(*_case([], [g]))
    assert np.isnan(ap) and ov.shape == (1, 0) and ov.dtype == np.float64
    ap, _, _, ov = eo.compute_ap(*_case([g], []))
    assert ap == 0 and ov.shape == (0, 1)
    gt_match, pred_match, _ = eo.compute_matches(*_case([g], []))
    assert gt_match.tolist() == [-1] and pred_match.size == 0


def test_trim_zeros_truncates_the_masks_not_the_rows():
    """A zero gt box in the middle: upstream drops the row but keeps the FIRST masks, so the
    prediction equal to the last mask finds nothing."""
    g0, g1, g2 = (_square(16, 16, 0, 0, 4, 4), _square(16, 16, 5, 5, 9, 9),
                  _square(16, 16, 10, 10, 14, 14))
    args = list(_case([g0, g1, g2], [g2]))
    args[0] = np.array([[1, 1, 2, 2], [0, 0, 0, 0], [3, 3, 4, 4]])
    gt_match, pred_match, ov = eo.compute_matches(*args)
    assert gt_match.tolist() == [-1, -1] and pred_match.tolist() == [-1] and ov.shape == (1, 2)


def closed_form_matches(overlaps, pred_cls, gt_cls, t, st):
    """What mrx_mask_matches computes: per prediction in rank order, among unmatched gts of its
    class whose IoU is NaN or >= both thresholds, the largest IoU (NaN above all, ties larger j)."""
    n, m = overlaps.shape
    gt_match, pred_match = -np.ones(m), -np.ones(n)
    tt, ss = comparison_threshold(t), comparison_threshold(st)
    for i in range(n):
        best = None
        for j in range(m):
            v = float(overlaps[i, j])
            if gt_match[j] > -1 or pred_cls[i] != gt_cls[j]:
                continue
            if not (np.isnan(v) or (v >= tt and v >= ss)):
                continue
            key = (2 if np.isnan(v) else 1, 0.0 if np.isnan(v) else v, j)
            best = key if best is None or key > best else best
        if best is not None:
            pred_match[i], gt_match[best[2]] = best[2], i
    return gt_match, pred_match


@pytest.mark.parametrize("seed", range(6))
def test_closed_form_equals_the_loop(seed):
    """Random overlaps with ties, NaNs and exact threshold values, both threshold kinds."""
    rng = np.random.default_rng(seed)
    n, m = rng.integers(1, 40, size=2)
    levels = np.array([0.0, 0.25, 0.5, 0.7, 0.75, 0.9, 1.0, np.nan], np.float32)
    ov = levels[rng.integers(0, len(levels), size=(n, m))]
    ov = np.where(rng.random((n, m)) < 0.3, rng.random((n, m)).astype(np.float32), ov)
    pc, gc = rng.integers(1, 3, size=n), rng.integers(1, 3, size=m)
    for t, st in [(0.5, 0.0), (np.float64(0.7), 0.0), (0.7, 0.0), (0.25, 0.5), (np.float64(0.75), np.float64(0.3))]:
        want = _loop_matches(ov, pc, gc, t, st)
        got = closed_form_matches(ov, pc, gc, t, st)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (t, st)


def _loop_matches(overlaps, pred_cls, gt_cls, iou_threshold, score_threshold):
    """The matching loop of eval_oracle.compute_matches on given overlaps (rows in rank order)."""
    n, m = overlaps.shape
    pred_match, gt_match = -np.ones(n), -np.ones(m)
    for i in range(n):
        sorted_ixs = np.argsort(overlaps[i], kind="stable")[::-1]
        low = np.where(overlaps[i, sorted_ixs] < score_threshold)[0]
        if low.size > 0:
            sorted_ixs = sorted_ixs[:low[0]]
        for j in sorted_ixs:
            if gt_match[j] > -1:
                continue
            if overlaps[i, j] < iou_threshold:
                break
            if pred_cls[i] == gt_cls[j]:
                gt_match[j], pred_match[i] = i, j
                break
    return gt_match, pred_match


@pytest.mark.parametrize("t", [0.5, 0.7, 0.75, 0.95, 1, 0, np.float64(0.7), np.float32(0.7),
                               np.float64(0.55), np.arange(0.5, 1.0, 0.05)[3]])
def test_comparison_threshold_orders_like_numpy(t):
    ious = np.float32(t) + np.array([-2, -1, 0, 1, 2], np.float32) * np.float32(2 ** -24)
    ious = np.concatenate([ious, np.nextafter(np.float32(t), np.float32([0, 2]))]).astype(np.float32)
    c = comparison_threshold(t)
    for v in ious:
        assert (float(v) < c) == bool(v < t), (t, v)


def test_comparison_threshold_refuses_other_types():
    with pytest.raises(TypeError):
        comparison_threshold("0.5")


@pytest.mark.parametrize("seed", range(4))
def test_ap_tail_equals_the_oracle(seed):
    rng = np.random.default_rng(seed)
    H, W = 24, 24
    m, n = int(rng.integers(0, 6)), int(rng.integers(0, 8))
    gt = [_square(H, W, *sorted(rng.integers(0, H, 2)), *sorted(rng.integers(0, W, 2)))
          for _ in range(m)]
    pred = [g.copy() for g in gt[:n]] + [_square(H, W, 0, 0, 5, 5)] * max(0, n - m)
    args = _case(gt, pred, gt_cls=rng.integers(1, 3, m), pred_cls=rng.integers(1, 3, len(pred)),
                 scores=rng.random(len(pred)))
    gt_match, pred_match, _ = eo.compute_matches(*args)
    want = eo.compute_ap(*args)
    got = evaluate.ap_from_matches(pred_match, gt_match)
    for a, b in zip(got, want[:3]):
        assert np.array_equal(a, b, equal_nan=True) and np.asarray(a).dtype == np.asarray(b).dtype
