"""CPU restatement of upstream's mask scoring (Matterport `mrcnn/utils.py`: `trim_zeros`,
`compute_overlaps_masks`, `compute_matches`, `compute_ap`, `compute_ap_range`), loop for loop.
TEST INFRASTRUCTURE ONLY.

*** PARITY UNPINNED ***  The reference does not vendor mrcnn/utils.py; these restate upstream's
published code.  The one stated difference: upstream's two `np.argsort` calls use the default
quicksort, which is unstable (introsort) above 16 elements, so the order of equal scores and
equal IoUs is implementation-defined there.  Here both use kind="stable" and are reversed, which
defines it: descending, NaN first, ties larger index first.
"""
import numpy as np


def trim_zeros(x):
    assert len(x.shape) == 2
    return x[~np.all(x == 0, axis=1)]


# One-line departures of the two orders and the loop below, each modelling a mutant of
# mrx_mask_matches' kernels (tools/mutate_eval.py): score ties by the smaller index first, NaN
# IoUs taken after every number (as if +0, still past both thresholds), a strict IoU threshold,
# and IoU ties to the smaller ground-truth index.
MATCH_VARIANTS = ("rank_tie_first", "nan_low", "thr_strict", "tie_small_j")


def score_order(pred_scores, variant=None):
    """compute_matches' prediction order: np.argsort(kind="stable") reversed -- descending, NaN
    first, equal scores larger index first."""
    s = np.asarray(pred_scores)
    if variant == "rank_tie_first":
        key = np.where(np.isnan(s), np.inf, s)
        return np.lexsort((np.arange(s.size), -key))
    return np.argsort(s, kind="stable")[::-1]


def match_loop(overlaps, pred_class_ids, gt_class_ids, iou_threshold=0.5, score_threshold=0.0,
               variant=None):
    """compute_matches' loop on overlaps [N, M] whose rows are the predictions in score order:
    (gt_match [M], pred_match [N]), float64, the rank of the matched prediction / the matched
    ground-truth index, or -1.  The thresholds compare as NumPy compares them with the IoU's
    dtype (NEP 50: a Python float weakly, in float32; a NumPy scalar strongly)."""
    pred_match = -1 * np.ones([overlaps.shape[0]])
    gt_match = -1 * np.ones([overlaps.shape[1]])
    for i in range(overlaps.shape[0]):
        row = overlaps[i]
        if variant == "nan_low":
            sorted_ixs = np.argsort(np.where(np.isnan(row), 0, row), kind="stable")[::-1]
            sorted_ixs = sorted_ixs[~(row[sorted_ixs] < score_threshold)]
        else:
            if variant == "tie_small_j":
                key = np.where(np.isnan(row), np.inf, row)
                sorted_ixs = np.lexsort((np.arange(row.size), -key))
            else:
                sorted_ixs = np.argsort(row, kind="stable")[::-1]
            low_score_idx = np.where(row[sorted_ixs] < score_threshold)[0]
            if low_score_idx.size > 0:
                sorted_ixs = sorted_ixs[:low_score_idx[0]]
        for j in sorted_ixs:
            if gt_match[j] > -1:
                continue
            iou = row[j]
            if iou < iou_threshold or (variant == "thr_strict" and iou == iou_threshold):
                if variant == "nan_low":
                    continue           # NaNs may still follow
                break
            if pred_class_ids[i] == gt_class_ids[j]:
                gt_match[j] = i
                pred_match[i] = j
                break
    return gt_match, pred_match


def compute_overlaps_masks(masks1, masks2):
    if masks1.shape[-1] == 0 or masks2.shape[-1] == 0:
        return np.zeros((masks1.shape[-1], masks2.shape[-1]))
    masks1 = np.reshape(masks1 > .5, (-1, masks1.shape[-1])).astype(np.float32)
    masks2 = np.reshape(masks2 > .5, (-1, masks2.shape[-1])).astype(np.float32)
    area1 = np.sum(masks1, axis=0)
    area2 = np.sum(masks2, axis=0)
    intersections = np.dot(masks1.T, masks2)
    union = area1[:, None] + area2[None, :] - intersections
    with np.errstate(invalid="ignore"):
        overlaps = intersections / union
    return overlaps


def compute_matches(gt_boxes, gt_class_ids, gt_masks, pred_boxes, pred_class_ids, pred_scores,
                    pred_masks, iou_threshold=0.5, score_threshold=0.0):
    gt_boxes = trim_zeros(gt_boxes)
    gt_masks = gt_masks[..., :gt_boxes.shape[0]]
    pred_boxes = trim_zeros(pred_boxes)
    pred_scores = pred_scores[:pred_boxes.shape[0]]
    indices = score_order(pred_scores)
    pred_boxes = pred_boxes[indices]
    pred_class_ids = pred_class_ids[indices]
    pred_scores = pred_scores[indices]
    pred_masks = pred_masks[..., indices]
    overlaps = compute_overlaps_masks(pred_masks, gt_masks)
    gt_match, pred_match = match_loop(overlaps, pred_class_ids, gt_class_ids[:gt_boxes.shape[0]],
                                      iou_threshold, score_threshold)
    return gt_match, pred_match, overlaps


def compute_ap(gt_boxes, gt_class_ids, gt_masks, pred_boxes, pred_class_ids, pred_scores,
               pred_masks, iou_threshold=0.5):
    gt_match, pred_match, overlaps = compute_matches(
        gt_boxes, gt_class_ids, gt_masks, pred_boxes, pred_class_ids, pred_scores, pred_masks,
        iou_threshold)
    with np.errstate(divide="ignore", invalid="ignore"):
        precisions = np.cumsum(pred_match > -1) / (np.arange(len(pred_match)) + 1)
        recalls = np.cumsum(pred_match > -1).astype(np.float32) / len(gt_match)
    precisions = np.concatenate([[0], precisions, [0]])
    recalls = np.concatenate([[0], recalls, [1]])
    for i in range(len(precisions) - 2, -1, -1):
        precisions[i] = np.maximum(precisions[i], precisions[i + 1])
    indices = np.where(recalls[:-1] != recalls[1:])[0] + 1
    mAP = np.sum((recalls[indices] - recalls[indices - 1]) * precisions[indices])
    return mAP, precisions, recalls, overlaps


def compute_ap_range(gt_box, gt_class_id, gt_mask, pred_box, pred_class_id, pred_score,
                     pred_mask, iou_thresholds=None, verbose=1):
    iou_thresholds = iou_thresholds if iou_thresholds is not None else np.arange(0.5, 1.0, 0.05)
    AP = []
    for iou_threshold in iou_thresholds:
        ap, precisions, recalls, overlaps = compute_ap(
            gt_box, gt_class_id, gt_mask, pred_box, pred_class_id, pred_score, pred_mask,
            iou_threshold=iou_threshold)
        if verbose:
            print("AP @{:.2f}:\t {:.3f}".format(iou_threshold, ap))
        AP.append(ap)
    AP = np.array(AP).mean()
    if verbose:
        print("AP @{:.2f}-{:.2f}:\t {:.3f}".format(iou_thresholds[0], iou_thresholds[-1], AP))
    return AP
