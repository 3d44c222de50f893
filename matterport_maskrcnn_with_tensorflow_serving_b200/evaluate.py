"""Drop-ins for upstream's mask scoring in `mrcnn.utils` (Matterport): `compute_overlaps_masks`,
`compute_matches`, `compute_ap` and `compute_ap_range`, with upstream's signatures, defaults and
return dtypes; NumPy in, NumPy out.  The mask IoUs and the matching run on the device
(`mrx_mask_extents`, `mrx_mask_overlaps`, `mrx_mask_matches`, DESIGN.md section 3.13): the masks
are bit-packed there and only the [N, M] overlaps and the matches come back.  `trim_zeros`, the
`> .5` threshold of non-bool masks and the AP tail run on the host, as upstream writes them.

The one difference from upstream: both of its `np.argsort` calls use the default, unstable
quicksort, so the order of equal scores and equal IoUs is implementation-defined there.  Here it
is what a stable sort reversed gives: descending, NaN first, ties larger index first.  Overlaps
equal NumPy's bit for bit while H*W <= 2^24; above that NumPy's float32 sums stop counting and
the device rounds the exact counts once each.
"""
from __future__ import annotations

import numpy as np

from . import _native as N
from .engine import MaskBatch, mask_matches, mask_overlaps


def trim_zeros(x):
    """[UPSTREAM] the rows of x that are not all zeros."""
    assert len(x.shape) == 2
    return x[~np.all(x == 0, axis=1)]


def ap_from_matches(pred_match, gt_match):
    """[UPSTREAM compute_ap, after compute_matches] (mAP, precisions, recalls) of one threshold's
    matches, upstream's NumPy lines as they are (M = 0 gives NaN with NumPy's warnings
    silenced)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        precisions = np.cumsum(pred_match > -1) / (np.arange(len(pred_match)) + 1)
        recalls = np.cumsum(pred_match > -1).astype(np.float32) / len(gt_match)
    precisions = np.concatenate([[0], precisions, [0]])
    recalls = np.concatenate([[0], recalls, [1]])
    for i in range(len(precisions) - 2, -1, -1):
        precisions[i] = np.maximum(precisions[i], precisions[i + 1])
    indices = np.where(recalls[:-1] != recalls[1:])[0] + 1
    mAP = np.sum((recalls[indices] - recalls[indices - 1]) * precisions[indices])
    return mAP, precisions, recalls


def _single_image_batch(class_ids, masks):
    import torch

    N.require_cuda()
    H, W = masks.shape[:2]
    return MaskBatch(N.load(), torch.device("cuda", torch.cuda.current_device()),
                     [[H, W, H, W, 0, 0, H, W]], [class_ids], [masks])


def _check_pair(masks1, masks2):
    if masks1.ndim != 3 or masks2.ndim != 3 or masks1.shape[:2] != masks2.shape[:2]:
        raise ValueError(f"masks must be [H, W, N] and [H, W, M], got {masks1.shape} and "
                         f"{masks2.shape}")


def compute_overlaps_masks(masks1, masks2):
    """IoU overlaps between two sets of masks [H, W, N] and [H, W, M]: float32 [N, M] (float64
    zeros when either set is empty)."""
    masks1, masks2 = np.asarray(masks1), np.asarray(masks2)
    if masks1.shape[-1] == 0 or masks2.shape[-1] == 0:
        return np.zeros((masks1.shape[-1], masks2.shape[-1]))
    _check_pair(masks1, masks2)
    a = _single_image_batch(np.zeros(masks1.shape[2], np.int32), masks1)
    b = _single_image_batch(np.zeros(masks2.shape[2], np.int32), masks2)
    return mask_overlaps(N.load(), a.planes, b.planes, a.d_geom, 1)[0].cpu().numpy()


def _matches(gt_boxes, gt_class_ids, gt_masks, pred_boxes, pred_class_ids, pred_scores,
             pred_masks, thresholds, score_threshold):
    """compute_matches for every threshold in one device pass: (gt_match [T, M], pred_match
    [T, N], overlaps) as upstream returns them per threshold."""
    import torch

    gt_boxes = trim_zeros(np.asarray(gt_boxes))
    gt_masks = np.asarray(gt_masks)[..., :gt_boxes.shape[0]]
    pred_boxes = trim_zeros(np.asarray(pred_boxes))
    pred_scores = np.asarray(pred_scores)[:pred_boxes.shape[0]]
    n, m = pred_boxes.shape[0], gt_boxes.shape[0]
    T = len(thresholds)
    if n == 0 or m == 0:
        return -np.ones((T, m)), -np.ones((T, n)), np.zeros((n, m))
    pred_masks = np.asarray(pred_masks)[..., :n]
    _check_pair(pred_masks, gt_masks)
    pred = _single_image_batch(np.asarray(pred_class_ids)[:n], pred_masks)
    gt = _single_image_batch(np.asarray(gt_class_ids)[:m], gt_masks)
    lib = N.load()
    d_ov = mask_overlaps(lib, pred.planes, gt.planes, pred.d_geom, 1)
    d_scores = torch.from_numpy(pred_scores.astype(np.float64).reshape(1, n)).to(d_ov.device)
    d_order, d_pm, d_gm = mask_matches(lib, d_ov, pred.d_counts, pred.d_class_ids, d_scores,
                                       N.MRX_F64, gt, thresholds, score_threshold)
    order = d_order[0].cpu().numpy()
    return (d_gm[:, 0].cpu().numpy().astype(np.float64),
            d_pm[:, 0].cpu().numpy().astype(np.float64), d_ov[0].cpu().numpy()[order])


def compute_matches(gt_boxes, gt_class_ids, gt_masks, pred_boxes, pred_class_ids, pred_scores,
                    pred_masks, iou_threshold=0.5, score_threshold=0.0):
    """Finds matches between prediction and ground truth instances.  Returns gt_match [M] and
    pred_match [N] (float64: the index of the matched instance or -1; predictions in
    descending score order) and overlaps [N, M] (rows in that order)."""
    gm, pm, overlaps = _matches(gt_boxes, gt_class_ids, gt_masks, pred_boxes, pred_class_ids,
                                pred_scores, pred_masks, [iou_threshold], score_threshold)
    return gm[0], pm[0], overlaps


def compute_ap(gt_boxes, gt_class_ids, gt_masks, pred_boxes, pred_class_ids, pred_scores,
               pred_masks, iou_threshold=0.5):
    """Average precision at one IoU threshold: (mAP, precisions, recalls, overlaps)."""
    gt_match, pred_match, overlaps = compute_matches(
        gt_boxes, gt_class_ids, gt_masks, pred_boxes, pred_class_ids, pred_scores, pred_masks,
        iou_threshold)
    return ap_from_matches(pred_match, gt_match) + (overlaps,)


def compute_ap_range(gt_box, gt_class_id, gt_mask, pred_box, pred_class_id, pred_score,
                     pred_mask, iou_thresholds=None, verbose=1):
    """The mean of compute_ap over iou_thresholds (default np.arange(0.5, 1.0, 0.05)), all
    thresholds matched in one device pass; prints upstream's lines when verbose."""
    iou_thresholds = iou_thresholds if iou_thresholds is not None else np.arange(0.5, 1.0, 0.05)
    gm, pm, _ = _matches(gt_box, gt_class_id, gt_mask, pred_box, pred_class_id, pred_score,
                         pred_mask, list(iou_thresholds), 0.0)
    AP = []
    for t, iou_threshold in enumerate(iou_thresholds):
        ap = ap_from_matches(pm[t], gm[t])[0]
        if verbose:
            print("AP @{:.2f}:\t {:.3f}".format(iou_threshold, ap))
        AP.append(ap)
    AP = np.array(AP).mean()
    if verbose:
        print("AP @{:.2f}-{:.2f}:\t {:.3f}".format(iou_thresholds[0], iou_thresholds[-1], AP))
    return AP
