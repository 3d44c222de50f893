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

`COCOevalSegm` is pycocotools' COCOeval for iouType "segm" (COCO mask AP) as a streaming
evaluator: the IoUs and matching of `evaluate()` run on the device as each batch is added
(`mrx_coco_ranks`, `mrx_coco_ious`, `mrx_coco_match`, DESIGN.md section 3.15); `accumulate()` and
`summarize()` run on the host and equal pycocotools' exactly.  `COCOevalBbox` is the same for
iouType "bbox" (COCO box AP): box IoUs and matching on the device (`mrx_coco_box_ious`,
`mrx_coco_match_f64area`, DESIGN.md section 3.17), no mask involved.  `COCOevalBoundary` is
boundary_iou_api's COCOeval for iouType "boundary" (Boundary AP): `COCOevalSegm` with the IoU
taken as the smaller of the mask IoU and the boundary IoU, the boundaries made on the device
(`mrx_mask_boundary`, `mrx_coco_boundary_ious`, DESIGN.md section 3.18).

`LVISEvalSegm` and `LVISEvalBbox` are lvis-api's LVISEval for "segm" and "bbox" (LVIS mask and box
AP, with APr / APc / APf) as streaming evaluators on the same device steps: `mrx_lvis_ranks` keeps
the first `max_dets` results of each image and only the categories the image is federated for,
DESIGN.md section 3.19.

`ann_to_mask` is Matterport's `CocoDataset.annToMask`, rasterised on the device (DESIGN.md
section 3.16).
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np

from . import _native as N
from .engine import (MaskBatch, Predictions, check_dilation_ratio, coco_boundary_evaluate_batch,
                     coco_box_evaluate_batch, coco_device_params, coco_evaluate_batch,
                     lvis_device_params, mask_matches, mask_overlaps)


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


# ----------------------------------------------------------------------------- COCO mask AP
class Params:
    """COCOeval's parameters for iouType "segm" or "bbox", with pycocotools' attribute names and
    defaults.
    `imgIds` is the sorted ids of the images added so far (it may be set to a subset before
    `accumulate`); `catIds` is the sorted category ids of the ground truth added so far unless
    given.  Only `useCats = 1` is supported."""

    def __init__(self, cat_ids=None, iou_thrs=None, rec_thrs=None, max_dets=(1, 10, 100),
                 area_rng=None, area_rng_lbl=None, iou_type="segm"):
        self.imgIds = []
        self.catIds = [] if cat_ids is None else sorted(set(int(c) for c in cat_ids))
        self.iouThrs = (np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
                        if iou_thrs is None else np.asarray(iou_thrs, dtype=np.float64))
        self.recThrs = (np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
                        if rec_thrs is None else np.asarray(rec_thrs, dtype=np.float64))
        self.maxDets = sorted(int(m) for m in max_dets)
        self.areaRng = ([[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2],
                         [96 ** 2, 1e5 ** 2]] if area_rng is None else
                        [[float(lo), float(hi)] for lo, hi in area_rng])
        self.areaRngLbl = (["all", "small", "medium", "large"] if area_rng_lbl is None
                           else list(area_rng_lbl))
        if len(self.areaRngLbl) != len(self.areaRng):
            raise ValueError(f"{len(self.areaRngLbl)} area labels for {len(self.areaRng)} ranges")
        self.useCats = 1
        self.iouType = iou_type


def _curves(score, matched, ignored, npig, rec_thrs):
    """accumulate's curves of one category from its detections in accumulate's order (score
    [n], matched and ignored [A, T, n]) and npig [A], its non-ignored ground truth per area range:
    for every area range a with npig[a] > 0, (a, recall [T] (the last recall, 0 without
    detections), precision [T, R] and scores [T, R] at rec_thrs).  Cumulative sums of the flags, a
    running maximum for the precision envelope and searchsorted, bit-equal to pycocotools' and
    lvis-api's loops."""
    nd = score.size
    T, R = matched.shape[1], len(rec_thrs)
    tp_sum = np.cumsum(matched & ~ignored, axis=2).astype(dtype=float)
    fp_sum = np.cumsum(~matched & ~ignored, axis=2).astype(dtype=float)
    eps = np.spacing(1)
    for a in range(matched.shape[0]):
        if npig[a] == 0:
            continue
        tp, fp = tp_sum[a], fp_sum[a]
        rc = tp / npig[a]
        pr = tp / (fp + tp + eps)
        last = rc[:, -1] if nd else 0
        pr = np.maximum.accumulate(pr[:, ::-1], axis=1)[:, ::-1]
        q = np.zeros((T, R))
        ss = np.zeros((T, R))
        for t in range(T):
            inds = np.searchsorted(rc[t], rec_thrs, side="left")
            hit = inds < nd
            q[t, hit] = pr[t, inds[hit]]
            ss[t, hit] = score[inds[hit]]
        yield a, last, q, ss


class _COCOevalBase:
    """What `COCOevalSegm` and `COCOevalBbox` share: the parameters, the category and image maps,
    the per-detection records each batch appends (`_record`), and pycocotools' `evaluate`,
    `accumulate` and `summarize` over them, which do not depend on the IoU type."""

    _iou_type = None

    def __init__(self, cat_ids=None, iou_thrs=None, rec_thrs=None, max_dets=(1, 10, 100),
                 area_rng=None, area_rng_lbl=None):
        self.params = Params(cat_ids, iou_thrs, rec_thrs, max_dets, area_rng, area_rng_lbl,
                             self._iou_type)
        coco_device_params(self.params)        # raises outside the kernels' limits
        self._init_records({}, cat_ids is None)
        self.stats = None

    def _init_records(self, cat_index, auto_cats):
        """The state every evaluator starts from, COCO or LVIS: the category and image maps, no
        records, parameters not yet frozen."""
        self._cat_index = cat_index   # category id -> dense index used on the device
        self._auto_cats = auto_cats
        self._frozen = None
        self._gt_cats = set()
        self._img_index = {}          # image id -> position in add order
        self._dets = []               # per batch: (img, cat, rank, score, matched, ignored)
        self._gts = []                # per batch: (img, cat, not ignored [n, A])
        self.eval = {}

    # ------------------------------------------------------------------ adding batches
    def _dense(self, cat_id):
        return self._cat_index.setdefault(int(cat_id), len(self._cat_index))

    def _freeze(self):
        p = self.params
        key = (tuple(np.ravel(p.iouThrs).tolist()), tuple(np.ravel(p.areaRng).tolist()),
               int(p.maxDets[-1]))
        if self._frozen is None:
            self._frozen = key
        elif key != self._frozen:
            raise ValueError("iouThrs, areaRng and maxDets[-1] changed after the first batch")
        coco_device_params(p)

    def _new_images(self, image_ids, n_items, gt_anns, what):
        if len(image_ids) != n_items:
            raise ValueError(f"{n_items} {what} but {len(image_ids)} image ids")
        if len(gt_anns) != len(image_ids):
            raise ValueError(f"{len(gt_anns)} ground-truth annotation lists for {len(image_ids)} "
                             "images")
        seen = set()
        for i in image_ids:
            if i in self._img_index or i in seen:
                raise ValueError(f"image {i!r} was already added")
            seen.add(i)

    # A batch takes these steps, run by add_results or, around one unmold for several evaluators,
    # by api_utils.unmold_coco_eval_batch: `_gt_tables` (host checks and the tables (cats, crowd,
    # area, segmentations or boxes), before anything is uploaded; `_batch_tables` for model
    # outputs, None for an empty batch), `_batch_status`, `_ground_truth`, `_ious` (the scorer on
    # `Predictions`: the engine's, after the packed expand when `_needs_masks`, or decoded
    # results) and `_record`
    _needs_masks = False

    def _batch_tables(self, items, image_ids, gt_anns):
        self._new_images(image_ids, len(items), gt_anns, "items")
        self._freeze()
        if len(items) == 0:
            return None
        return self._gt_tables(image_ids, gt_anns, [(int(it[2][0]), int(it[2][1]))
                                                    for it in items])

    def _batch_status(self, image_ids, gt_cats):
        """The batch's LVIS status table, which its IoU step and `_record` read; None for COCO."""
        return None

    def _ground_truth(self, lib, device, geoms, tables):
        """(None, tables): box ground truth goes up inside the scorer."""
        return None, tables

    @staticmethod
    def _by_image(results, image_ids, check):
        """results as one list per image of image_ids, each result k replaced by check(k, r),
        which raises for a result it does not take."""
        pos = {i: b for b, i in enumerate(image_ids)}
        dets = [[] for _ in image_ids]
        for k, r in enumerate(results):
            if r.get("image_id") not in pos:
                raise ValueError(f"result {k}: image {r.get('image_id')!r} is not one of the "
                                 "batch's image ids")
            dets[pos[r["image_id"]]].append(check(k, r))
        return dets

    def _class_map(self, C, category_ids):
        """int32 [C]: the engine's class id -> dense category (-1 where category_ids has none)."""
        class_map = np.full(C, -1, np.int32)
        for c in range(C):
            try:
                class_map[c] = self._dense(c if category_ids is None else category_ids[c])
            except (IndexError, KeyError):
                pass
        return class_map

    @staticmethod
    def _where(image_id, k, ann):
        return f"image {image_id!r}, annotation {k}" + (
            f" (id {ann['id']!r})" if isinstance(ann, dict) and "id" in ann else "")

    @staticmethod
    def _padded(rows, R, dtype, tail=()):
        out = np.zeros((len(rows), R) + tuple(tail), dtype)
        for b, r in enumerate(rows):
            if len(r):
                out[b, :len(r)] = r
        return out

    def _record(self, image_ids, res, gt_cats, gt_crowd, gt_area, status=None):
        """Append the per-detection records of one batch (`coco_evaluate_batch`'s dict) and the
        ground truth's non-ignored flags per area range.  status: `_batch_status`'s table."""
        first = len(self._img_index)
        for b, i in enumerate(image_ids):
            self._img_index[i] = first + b
        b, i = np.nonzero(res["keep"])
        self._dets.append((first + b, res["cat"][b, i], res["rank"][b, i], res["score"][b, i],
                           res["match"][:, :, b, i].transpose(2, 0, 1) > -1,
                           res["ignore"][:, :, b, i].transpose(2, 0, 1)))
        rng = np.asarray(self._area_rng(), np.float64).reshape(-1, 2)
        img = np.concatenate([np.full(len(c), first + b, np.int64) for b, c in enumerate(gt_cats)]
                             + [np.zeros(0, np.int64)])
        crowd = np.concatenate(gt_crowd + [np.zeros(0, np.uint8)]).astype(bool)
        area = np.concatenate(gt_area + [np.zeros(0)])
        nonig = ~crowd[:, None] & (area[:, None] >= rng[:, 0]) & (area[:, None] <= rng[:, 1])
        self._gts.append((img, np.concatenate(gt_cats + [np.zeros(0, np.int32)]), nonig))
        self._sync_params()

    def _area_rng(self):
        return self.params.areaRng

    def _sync_params(self):
        p = self.params
        p.imgIds = sorted(self._img_index)
        if self._auto_cats:
            p.catIds = sorted(self._gt_cats)

    # ------------------------------------------------------------------ pycocotools' API
    def evaluate(self):
        """pycocotools runs the per-image evaluation here; this evaluator has already run it on
        the device as each batch was added, so there is nothing left to do."""

    def accumulate(self):
        """pycocotools' accumulate over the images of `params.imgIds` (in sorted id order) and
        the categories of `params.catIds`, vectorised: per category one lexsort of its
        detections by (-score, image, rank), the maxDets cuts as masks, cumulative sums of the
        match flags, a running maximum for the precision envelope and searchsorted at
        `recThrs`.  Bit-equal to pycocotools' loop."""
        self._freeze()
        p = self.params
        img_ids = list(np.unique(p.imgIds)) if len(p.imgIds) else []
        cat_ids = list(np.unique(p.catIds)) if len(p.catIds) else []
        T, R, K = len(p.iouThrs), len(p.recThrs), len(cat_ids)
        A, M = len(p.areaRng), len(p.maxDets)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        scores = -np.ones((T, R, K, A, M))
        for k, npig, rank, score, matched, ignored in self._by_category(img_ids, cat_ids, A, T):
            for m, max_det in enumerate(p.maxDets):
                cut = rank < max_det
                for a, rc, q, ss in _curves(score[cut], matched[:, :, cut], ignored[:, :, cut],
                                            npig, p.recThrs):
                    recall[:, k, a, m] = rc
                    precision[:, :, k, a, m] = q
                    scores[:, :, k, a, m] = ss
        self.eval = {"params": p, "counts": [T, R, K, A, M], "precision": precision,
                     "recall": recall, "scores": scores}

    def _by_category(self, img_ids, cat_ids, A, T):
        """The records of the images of img_ids and the categories of cat_ids, per category
        position k that has non-ignored ground truth in some area range: (k, npig [A], the
        number of non-ignored instances per range, and its detections' rank, score, matched and
        ignored [A, T, n] in accumulate's order: one lexsort by (-score, image position in img_ids,
        rank within (image, category)))."""
        K = len(cat_ids)
        img_rank = np.full(len(self._img_index) + 1, -1, np.int64)   # add position -> img_ids
        for r, i in enumerate(img_ids):
            if i in self._img_index:
                img_rank[self._img_index[i]] = r
        cat_k = np.full(len(self._cat_index) + 1, -1, np.int64)   # dense -> cat_ids position
        for k, c in enumerate(cat_ids):
            if int(c) in self._cat_index:
                cat_k[self._cat_index[int(c)]] = k

        def cat(parts, i, empty):
            return np.concatenate([x[i] for x in parts] + [empty])

        d_img = img_rank[cat(self._dets, 0, np.zeros(0, np.int64))]
        d_k = cat_k[cat(self._dets, 1, np.zeros(0, np.int32))]
        d_rank = cat(self._dets, 2, np.zeros(0, np.int32))
        d_score = cat(self._dets, 3, np.zeros(0))
        d_tp = cat(self._dets, 4, np.zeros((0, A, T), bool))
        d_ig = cat(self._dets, 5, np.zeros((0, A, T), bool))
        g_img = img_rank[cat(self._gts, 0, np.zeros(0, np.int64))]
        g_k = cat_k[cat(self._gts, 1, np.zeros(0, np.int32))]
        g_nonig = cat(self._gts, 2, np.zeros((0, A), bool))
        npig = np.zeros((K + 1, A), np.int64)
        ok = (g_img >= 0) & (g_k >= 0)
        np.add.at(npig, g_k[ok], g_nonig[ok])
        ok = (d_img >= 0) & (d_k >= 0)
        d_img, d_k, d_rank, d_score, d_tp, d_ig = (x[ok] for x in (d_img, d_k, d_rank, d_score,
                                                                   d_tp, d_ig))
        by_k = np.argsort(d_k, kind="stable")
        bounds = np.searchsorted(d_k[by_k], np.arange(K + 1))
        for k in range(K):
            if not (npig[k] > 0).any():
                continue
            sel = by_k[bounds[k]:bounds[k + 1]]
            order = sel[np.lexsort((d_rank[sel], d_img[sel], -d_score[sel]))]
            yield (k, npig[k], d_rank[order], d_score[order], d_tp[order].transpose(1, 2, 0),
                   d_ig[order].transpose(1, 2, 0))

    def summarize(self):
        """pycocotools' twelve `stats` (each the mean of the entries > -1, or -1 if none), printed
        in its format."""
        if not self.eval:
            raise Exception("Please run accumulate() first")
        p = self.params

        def _summarize(ap=1, iouThr=None, areaRng="all", maxDets=100):
            iStr = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}"
            titleStr = "Average Precision" if ap == 1 else "Average Recall"
            typeStr = "(AP)" if ap == 1 else "(AR)"
            iouStr = "{:0.2f}:{:0.2f}".format(p.iouThrs[0], p.iouThrs[-1]) \
                if iouThr is None else "{:0.2f}".format(iouThr)
            aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
            s = self.eval["precision"] if ap == 1 else self.eval["recall"]
            if iouThr is not None:
                s = s[np.where(iouThr == p.iouThrs)[0]]
            s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
            mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
            print(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
            return mean_s

        md = p.maxDets
        stats = np.zeros((12,))
        stats[0] = _summarize(1)
        stats[1] = _summarize(1, iouThr=.5, maxDets=md[2])
        stats[2] = _summarize(1, iouThr=.75, maxDets=md[2])
        stats[3] = _summarize(1, areaRng="small", maxDets=md[2])
        stats[4] = _summarize(1, areaRng="medium", maxDets=md[2])
        stats[5] = _summarize(1, areaRng="large", maxDets=md[2])
        stats[6] = _summarize(0, maxDets=md[0])
        stats[7] = _summarize(0, maxDets=md[1])
        stats[8] = _summarize(0, maxDets=md[2])
        stats[9] = _summarize(0, areaRng="small", maxDets=md[2])
        stats[10] = _summarize(0, areaRng="medium", maxDets=md[2])
        stats[11] = _summarize(0, areaRng="large", maxDets=md[2])
        self.stats = stats


class COCOevalSegm(_COCOevalBase):
    """pycocotools' `COCOeval(cocoGt, cocoDt, "segm")` as a streaming evaluator: batches are added
    one at a time (`add_batch` with model outputs, `add_results` with COCO segm results), the
    per-image work of `evaluate()` -- mask IoUs and matching for every (image, category, area
    range, threshold) -- runs on the device as each batch arrives, and only compact
    per-detection records stay on the host.  `accumulate()` and `summarize()` then give
    pycocotools' `eval` arrays (`precision` and `scores` [T, R, K, A, M], `recall` [T, K, A, M],
    float64, -1 where undefined) and its twelve `stats`, exactly.

    Ground-truth annotations are COCO dicts: `category_id`, `segmentation` an RLE dict ({'size':
    [H, W], 'counts': compressed `str` / `bytes` or an uncompressed count list}) or, with
    `polygons=True`, a polygon or box list as a COCO instances file holds every non-crowd
    annotation (rasterised on the device as pycocotools' annToRLE does, `MaskBatch.from_coco`),
    `iscrowd`
    (default 0; a crowd region's IoU is intersection / detection area, it absorbs any number of
    detections and never counts as a miss), and `area` (the annotation's area, which decides its
    area range; a detection's area is its mask's pixel count).

    Stated differences from pycocotools: matches are recorded by position, where pycocotools
    stores annotation ids and tests them for truth (so an annotation with id 0 counts as
    unmatched there); a ground-truth dict without `area` gets its mask's pixel count, where
    pycocotools raises KeyError; with the default `polygons=False`, polygon segmentations
    raise ValueError (rasterise them to RLE first).  Detections are RLE only, with or without
    `polygons`.  `iouThrs`, `areaRng` and `maxDets[-1]` are used on the device as each batch is
    added, so they must not change after the first batch."""

    _iou_type = "segm"

    def __init__(self, cat_ids=None, iou_thrs=None, rec_thrs=None, max_dets=(1, 10, 100),
                 area_rng=None, area_rng_lbl=None, polygons=False):
        super().__init__(cat_ids, iou_thrs, rec_thrs, max_dets, area_rng, area_rng_lbl)
        self._polygons = bool(polygons)

    def _gt_tables(self, image_ids, gt_anns, shapes):
        """Per image: dense category ids, crowd flags, areas (NaN where absent) and segmentations
        (RLE dicts, and polygon or box lists when the evaluator takes them), each annotation
        checked."""
        cats, crowd, area, rles = [], [], [], []
        for image_id, anns, hw in zip(image_ids, gt_anns, shapes):
            c, cr, ar, rl = [], [], [], []
            for k, ann in enumerate(anns):
                where = self._where(image_id, k, ann)
                seg = ann.get("segmentation") if isinstance(ann, dict) else None
                if isinstance(seg, list) and not self._polygons:
                    raise ValueError(f"{where}: polygon segmentations are not supported; give "
                                     "the mask as RLE")
                if isinstance(seg, list):
                    pass                   # checked by pack_polygons, naming the instance
                elif not isinstance(seg, dict) or "counts" not in seg or "size" not in seg:
                    raise ValueError(f"{where}: segmentation must be an RLE dict with 'size' and "
                                     "'counts'")
                if isinstance(seg, dict):
                    size = [int(v) for v in np.ravel(seg["size"])]
                    if hw is not None and size != list(hw):
                        raise ValueError(f"{where}: RLE size {size} is not the image's "
                                         f"{list(hw)}")
                cat = int(ann["category_id"])
                self._gt_cats.add(cat)
                c.append(self._dense(cat))
                cr.append(1 if ann.get("iscrowd", 0) else 0)
                ar.append(float(ann["area"]) if "area" in ann else np.nan)
                rl.append(seg)
            cats.append(np.asarray(c, np.int32))
            crowd.append(np.asarray(cr, np.uint8))
            area.append(np.asarray(ar, np.float64))
            rles.append(rl)
        return cats, crowd, area, rles

    def _ground_truth(self, lib, device, geoms, tables):
        """The batch's ground truth decoded on the device (a `MaskBatch` of geoms), and tables
        with each missing area replaced by its mask's pixel count."""
        cats, crowd, area, segs = tables
        gt = (MaskBatch.from_coco if self._polygons else MaskBatch.from_rle)(lib, device, geoms,
                                                                            cats, segs)
        if any(np.isnan(a).any() for a in area):
            mask_area = gt.planes.d_areas.cpu().numpy()
            area = [np.where(np.isnan(a), mask_area[b, :len(a)], a) for b, a in enumerate(area)]
        return gt, (cats, crowd, area, segs)

    def _ious(self, lib, pred, gt, tables, class_map, status):
        """The IoU step, the one part a mask IoU type replaces: the scorer's dict of pred (with
        planes) against gt."""
        _, crowd, area, _ = tables
        return coco_evaluate_batch(lib, pred.planes, pred.class_ids, pred.scores, gt,
                                   self._padded(crowd, gt.R, np.uint8),
                                   self._padded(area, gt.R, np.float64), class_map, self.params,
                                   status=status)

    def add_batch(self, items, image_ids, gt_anns, category_ids=None):
        """Evaluate model outputs against COCO ground truth: items as for
        `api_utils.unmold_detections_batch`, one image id and one list of annotation dicts per
        item.  The kept instances are expanded straight to packed planes on the device
        (`enqueue_packed`; no mask or RLE is made), the annotations are decoded there
        (`MaskBatch.from_rle`), and `category_ids` maps class ids to category ids as in
        `unmold_coco_results_batch` (None keeps the class id).  With `polygons=True` the
        annotations may be polygon or box lists, rasterised there (`MaskBatch.from_coco`)."""
        from . import api_utils

        api_utils.unmold_coco_eval_batch(items, image_ids, gt_anns, [self], category_ids)

    _needs_masks = True

    def add_results(self, results, gt_anns, image_ids, image_shapes=None):
        """Evaluate COCO segm results -- dicts {'image_id', 'category_id', 'score',
        'segmentation': RLE dict} as `loadRes` takes them and `unmold_coco_results_batch`
        returns them -- against gt_anns[b], the annotation dicts of image_ids[b].  Every result's
        image must be one of image_ids.  Both sides are decoded on the device; an image's shape
        is its RLEs' size, or image_shapes[b] = (height, width) when given (the RLEs must agree
        with it).  An image whose ground truth has polygons (`polygons=True`) and no RLE at all
        has no size to take, so it needs image_shapes; without it this raises ValueError."""
        import torch

        self._new_images(image_ids, len(gt_anns), gt_anns, "annotation lists")
        if image_shapes is not None and len(image_shapes) != len(image_ids):
            raise ValueError(f"{len(image_shapes)} image shapes for {len(image_ids)} images")
        self._freeze()
        if len(image_ids) == 0:
            return

        def check(k, r):
            seg = r.get("segmentation")
            if not isinstance(seg, dict) or "counts" not in seg or "size" not in seg:
                raise ValueError(f"result {k}: segmentation must be an RLE dict with 'size' and "
                                 "'counts'")
            return r

        dets = self._by_image(results, image_ids, check)
        shapes = []
        for image_id, d, anns in zip(image_ids, dets, gt_anns):
            sizes = {tuple(int(v) for v in np.ravel(x["segmentation"]["size"])) for x in d}
            sizes |= {tuple(int(v) for v in np.ravel(a["segmentation"]["size"])) for a in anns
                      if isinstance(a, dict) and isinstance(a.get("segmentation"), dict)
                      and "size" in a["segmentation"]}
            if image_shapes is not None:
                sizes.add(tuple(int(v) for v in image_shapes[len(shapes)]))
            if len(sizes) > 1:
                raise ValueError(f"image {image_id!r}: RLE sizes {sorted(sizes)} differ")
            if not sizes and self._polygons and any(isinstance(a, dict) and isinstance(a.get("segmentation"), list)
                                 for a in anns):
                raise ValueError(f"image {image_id!r}: its ground truth is polygons only, so its "
                                 "shape is unknown; give it in image_shapes")
            shapes.append(sizes.pop() if sizes else (1, 1))
        tables = self._gt_tables(image_ids, gt_anns, shapes)
        status = self._batch_status(image_ids, tables[0])
        N.require_cuda()
        lib = N.load()
        dev = torch.device("cuda", torch.cuda.current_device())
        geoms = [[H, W, H, W, 0, 0, H, W] for H, W in shapes]
        pred_cls = [np.asarray([self._dense(x["category_id"]) for x in d], np.int32) for d in dets]
        pred = MaskBatch.from_rle(lib, dev, geoms, pred_cls, [[x["segmentation"] for x in d]
                                                              for d in dets])
        gt, tables = self._ground_truth(lib, dev, geoms, tables)
        scores = self._padded([[float(x["score"]) for x in d] for d in dets], pred.R, np.float64)
        res = self._ious(lib, Predictions(pred.d_counts, pred.d_class_ids,
                                          torch.from_numpy(scores).to(dev), pred.d_regions,
                                          pred.planes),
                         gt, tables, np.arange(max(len(self._cat_index), 1), dtype=np.int32),
                         status)
        self._record(image_ids, res, *tables[:3], status)


class COCOevalBoundary(COCOevalSegm):
    """boundary_iou_api's `COCOeval(cocoGt, cocoDt, "boundary", dilation_ratio)` (Boundary AP,
    Cheng et al., "Boundary IoU", CVPR 2021) as a streaming evaluator: `COCOevalSegm` with only
    the IoU step replaced.  A pair's IoU is the smaller of its mask IoU and the IoU of the two
    masks' boundaries (mask AND NOT mask eroded by a (2d+1) x (2d+1) square, nothing outside the
    image; d = max(1, round(dilation_ratio * image diagonal)) per image), both with the crowd rule
    (a crowd's union is the detection's mask or boundary area).  The boundaries are made on the
    device from the packed planes (`mrx_mask_boundary`, DESIGN.md section 3.18) and both IoUs come
    from one walk over the pair (`mrx_coco_boundary_ious`); areas, ranges, matching,
    `accumulate()` and `summarize()` are segm's.

    `dilation_ratio` must be a finite number > 0 (else ValueError) and, like `iouThrs`, must not
    change after the first batch; it is `params.dilation_ratio`.  The stated differences from
    pycocotools are `COCOevalSegm`'s."""

    _iou_type = "boundary"

    def __init__(self, cat_ids=None, iou_thrs=None, rec_thrs=None, max_dets=(1, 10, 100),
                 area_rng=None, area_rng_lbl=None, polygons=False, dilation_ratio=0.02):
        super().__init__(cat_ids, iou_thrs, rec_thrs, max_dets, area_rng, area_rng_lbl, polygons)
        self.params.dilation_ratio = check_dilation_ratio(dilation_ratio)
        self._frozen_ratio = None

    def _freeze(self):
        super()._freeze()
        r = check_dilation_ratio(self.params.dilation_ratio)
        if self._frozen_ratio is None:
            self._frozen_ratio = r
        elif r != self._frozen_ratio:
            raise ValueError("dilation_ratio changed after the first batch")

    def _ious(self, lib, pred, gt, tables, class_map, status):
        _, crowd, area, _ = tables
        return coco_boundary_evaluate_batch(lib, pred.planes, pred.boxes, pred.class_ids,
                                            pred.scores, gt, self._padded(crowd, gt.R, np.uint8),
                                            self._padded(area, gt.R, np.float64), class_map,
                                            self.params, self._frozen_ratio)


class COCOevalBbox(_COCOevalBase):
    """pycocotools' `COCOeval(cocoGt, cocoDt, "bbox")` as a streaming evaluator, with
    `COCOevalSegm`'s API: `add_batch` with model outputs, `add_results` with COCO bbox results,
    then `accumulate()` and `summarize()` give pycocotools' `eval` arrays and twelve `stats`
    exactly.  The per-image work of `evaluate()` -- bbIou, bit for bit, and the matching for every
    (image, category, area range, threshold) -- runs on the device as each batch arrives; no mask
    is made or read.

    Ground-truth annotations are COCO dicts with `category_id`, `bbox` ([x, y, w, h]), `area`
    (which decides the area range) and `iscrowd` (default 0; a crowd box's IoU is intersection /
    detection area).  `segmentation` is not read.  A detection's area is w*h of its box, as
    `loadRes` stores it for bbox results.

    Stated differences from pycocotools: matches are recorded by position, as in `COCOevalSegm`;
    an annotation without `bbox` or `area` raises ValueError where pycocotools raises KeyError; a
    `bbox` that is not 4 numbers, or whose x, y, w, h, x + w, y + h or w * h is not finite, and a
    NaN `area`, raise ValueError (pycocotools computes NaN IoUs from such boxes, which its loop
    takes as matches).  `iouThrs`, `areaRng` and `maxDets[-1]` must not change after the first
    batch."""

    _iou_type = "bbox"

    @staticmethod
    def _box(bb, where):
        """bb as float64 [4], checked: 4 numbers, and x, y, w, h, x+w, y+h, w*h all finite."""
        try:
            box = np.asarray(bb, dtype=np.float64)
        except (TypeError, ValueError):
            box = None
        if box is None or box.shape != (4,):
            raise ValueError(f"{where}: bbox must be 4 numbers [x, y, w, h], got {bb!r}")
        with np.errstate(over="ignore", invalid="ignore"):
            derived = np.array([box[0] + box[2], box[1] + box[3], box[2] * box[3]])
        if not (np.isfinite(box).all() and np.isfinite(derived).all()):
            raise ValueError(f"{where}: bbox {bb!r} is not finite (its x, y, w, h, x+w, y+h and "
                             "w*h must be)")
        return box

    def _gt_tables(self, image_ids, gt_anns, shapes=None):
        """Per image: dense category ids, crowd flags, areas and boxes [M, 4], each annotation
        checked (the image shapes are not needed)."""
        cats, crowd, area, boxes = [], [], [], []
        for image_id, anns in zip(image_ids, gt_anns):
            c, cr, ar, bx = [], [], [], []
            for k, ann in enumerate(anns):
                where = self._where(image_id, k, ann)
                for key in ("bbox", "area"):
                    if not isinstance(ann, dict) or key not in ann:
                        raise ValueError(f"{where}: no '{key}'")
                bx.append(self._box(ann["bbox"], where))
                a = float(ann["area"])
                if np.isnan(a):
                    raise ValueError(f"{where}: area is NaN")
                cat = int(ann["category_id"])
                self._gt_cats.add(cat)
                c.append(self._dense(cat))
                cr.append(1 if ann.get("iscrowd", 0) else 0)
                ar.append(a)
            cats.append(np.asarray(c, np.int32))
            crowd.append(np.asarray(cr, np.uint8))
            area.append(np.asarray(ar, np.float64))
            boxes.append(np.asarray(bx, np.float64).reshape(-1, 4))
        return cats, crowd, area, boxes

    def _gt_arrays(self, tables):
        """The padded host arrays of coco_box_evaluate_batch's ground truth."""
        cats, crowd, area, boxes = tables
        R2 = max(max((len(c) for c in cats), default=0), 1)
        return (np.asarray([len(c) for c in cats], np.int32), self._padded(cats, R2, np.int32),
                self._padded(boxes, R2, np.float64, (4,)), self._padded(crowd, R2, np.uint8),
                self._padded(area, R2, np.float64))

    def _ious(self, lib, pred, gt, tables, class_map, status):
        """The scorer's dict of pred (boxes, no planes) against the tables' boxes (gt is None)."""
        return coco_box_evaluate_batch(lib, pred.boxes, pred.counts, pred.class_ids, pred.scores,
                                       *self._gt_arrays(tables), class_map, self.params,
                                       status=status)

    def add_batch(self, items, image_ids, gt_anns, category_ids=None):
        """Evaluate model outputs against COCO ground truth: items as for
        `api_utils.unmold_detections_batch`, one image id and one list of annotation dicts per
        item, `category_ids` as in `unmold_coco_results_batch` (None keeps the class id).  Only
        the unmold prepare step runs (`enqueue(..., expand=False)`): the kept boxes are scored
        where it leaves them, and no mask is expanded."""
        from . import api_utils

        api_utils.unmold_coco_eval_batch(items, image_ids, gt_anns, [self], category_ids)

    def add_results(self, results, gt_anns, image_ids):
        """Evaluate COCO bbox results -- dicts {'image_id', 'category_id', 'score', 'bbox':
        [x, y, w, h]} as `loadRes` takes them and `unmold_coco_results_batch` returns them --
        against gt_anns[b], the annotation dicts of image_ids[b].  Every result's image must be
        one of image_ids.  No image shape is needed."""
        self._new_images(image_ids, len(gt_anns), gt_anns, "annotation lists")
        self._freeze()
        if len(image_ids) == 0:
            return

        def check(k, r):
            if "bbox" not in r:
                raise ValueError(f"result {k}: no 'bbox'")
            return self._box(r["bbox"], f"result {k}"), r

        dets = self._by_image(results, image_ids, check)
        tables = self._gt_tables(image_ids, gt_anns)
        status = self._batch_status(image_ids, tables[0])
        N.require_cuda()
        R1 = max(max(len(d) for d in dets), 1)
        pred = Predictions(
            np.asarray([len(d) for d in dets], np.int32),
            self._padded([[self._dense(r["category_id"]) for _, r in d] for d in dets], R1,
                         np.int32),
            self._padded([[float(r["score"]) for _, r in d] for d in dets], R1, np.float64),
            self._padded([[box for box, _ in d] for d in dets], R1, np.float64, (4,)))
        res = self._ious(N.load(), pred, None, tables,
                         np.arange(max(len(self._cat_index), 1), dtype=np.int32), status)
        self._record(image_ids, res, *tables[:3], status)


# ----------------------------------------------------------------------------- LVIS mask and box AP
class LVISParams:
    """LVISEval's parameters (lvis-api's `Params`, snake_case names and defaults): `iou_thrs`,
    `rec_thrs`, `area_rng` and `area_rng_lbl` as pycocotools', `max_dets` one int (300, the
    per-image cut of LVISResults), `img_count_lbl` ["r", "c", "f"], `use_cats` 1 (the only one
    supported).  `cat_ids` is the sorted ids of every category of the dataset unless given;
    `img_ids` is the sorted ids of the images added so far (either may be set to a subset before
    `accumulate`)."""

    def __init__(self, cat_ids, iou_thrs=None, rec_thrs=None, max_dets=300, area_rng=None,
                 area_rng_lbl=None, img_count_lbl=None, iou_type="segm"):
        coco = Params(cat_ids, iou_thrs, rec_thrs, (1,), area_rng, area_rng_lbl, iou_type)
        self.img_ids = []
        self.cat_ids = coco.catIds
        self.iou_thrs = coco.iouThrs
        self.rec_thrs = coco.recThrs
        self.max_dets = int(max_dets)
        self.area_rng = coco.areaRng
        self.area_rng_lbl = coco.areaRngLbl
        self.use_cats = 1
        self.img_count_lbl = ["r", "c", "f"] if img_count_lbl is None else list(img_count_lbl)
        self.iou_type = iou_type


_LVIS_IMAGE_KEYS = ("id", "height", "width", "neg_category_ids", "not_exhaustive_category_ids")


class _LVISeval:
    """What `LVISEvalSegm` and `LVISEvalBbox` add to the COCO evaluator of their IoU type (the
    class that follows this one in their bases): lvis-api's parameters, the per-batch status table
    of the federated filter, the not-exhaustive rule on the downloaded flags, and LVISEval's
    `accumulate`, `summarize` and `print_results` over the same records."""

    def __init__(self, categories, images, cat_ids=None, iou_thrs=None, rec_thrs=None,
                 max_dets=300, area_rng=None, area_rng_lbl=None, img_count_lbl=None):
        self._freq = {}
        for k, c in enumerate(categories):
            if not isinstance(c, dict) or "id" not in c or "frequency" not in c:
                raise ValueError(f"category {k}: needs 'id' and 'frequency'")
            self._freq[int(c["id"])] = c["frequency"]
        self.params = LVISParams(sorted(self._freq) if cat_ids is None else cat_ids, iou_thrs,
                                 rec_thrs, max_dets, area_rng, area_rng_lbl, img_count_lbl,
                                 self._iou_type)
        for c, f in self._freq.items():
            if f not in self.params.img_count_lbl:
                raise ValueError(f"category {c}: frequency {f!r} is not one of "
                                 f"{self.params.img_count_lbl}")
        unknown = [c for c in self.params.cat_ids if c not in self._freq]
        if unknown:
            raise ValueError(f"cat_ids {unknown[:5]} are not categories of the dataset")
        if not self.params.cat_ids:
            raise ValueError("no categories to evaluate")
        lvis_device_params(self.params)        # raises outside the kernels' limits
        self._images = {}
        for k, im in enumerate(images):
            missing = [key for key in _LVIS_IMAGE_KEYS
                       if not isinstance(im, dict) or key not in im]
            if missing:
                name = im.get("id", k) if isinstance(im, dict) else k
                raise ValueError(f"image {name!r}: no {missing}")
            self._images[im["id"]] = im
        # the dense category index is the position in the constructor's cat_ids, fixed for good
        self._init_records({c: k for k, c in enumerate(self.params.cat_ids)}, False)
        self.results = {}

    def _dense(self, cat_id):
        """The dense index of a category, -1 for one outside the constructor's cat_ids (its
        ground truth is not read and its detections are not evaluated, as in lvis-api)."""
        return self._cat_index.get(int(cat_id), -1)

    def _freeze(self):
        p = self.params
        key = (tuple(np.ravel(p.iou_thrs).tolist()), tuple(np.ravel(p.area_rng).tolist()),
               int(p.max_dets))
        if self._frozen is None:
            lvis_device_params(p)
            self._frozen = key
        elif key != self._frozen:
            raise ValueError("iou_thrs, area_rng and max_dets changed after the first batch")

    def _new_images(self, image_ids, n_items, gt_anns, what):
        for i in image_ids:
            if i not in self._images:
                raise ValueError(f"image {i!r} is not one of the dataset's images")
        super()._new_images(image_ids, n_items, gt_anns, what)

    def _gt_tables(self, image_ids, gt_anns, shapes=None):
        """The COCO evaluator's tables with every instance non-crowd (LVISEval's compute_iou
        passes iscrowd = 0), after the LVIS checks."""
        for image_id, anns, hw in zip(image_ids, gt_anns,
                                      shapes if shapes is not None else [None] * len(image_ids)):
            im = self._images[image_id]
            if hw is not None and tuple(hw) != (int(im["height"]), int(im["width"])):
                raise ValueError(f"image {image_id!r}: shape {tuple(hw)} is not its height and "
                                 f"width {(im['height'], im['width'])}")
            for k, ann in enumerate(anns):
                if isinstance(ann, dict) and ann.get("ignore"):
                    raise ValueError(f"{self._where(image_id, k, ann)}: 'ignore' annotations are "
                                     "not supported")
        cats, crowd, area, segs = super()._gt_tables(image_ids, gt_anns, shapes)
        return cats, [np.zeros_like(c) for c in crowd], area, segs

    def _batch_status(self, image_ids, gt_cats):
        return self.status_table(image_ids, gt_cats)

    def status_table(self, image_ids, gt_cats):
        """uint8 [n, K]: per image and dense category the MRX_LVIS_* bits, POSITIVE where
        gt_cats[b] (dense categories of image b's ground truth) has it, NEGATIVE where it is in
        the image's neg_category_ids, NOT_EXHAUSTIVE where it is in its
        not_exhaustive_category_ids."""
        status = np.zeros((len(image_ids), len(self._cat_index)), np.uint8)
        for b, (image_id, c) in enumerate(zip(image_ids, gt_cats)):
            im = self._images[image_id]
            c = np.asarray(c, np.int64)
            status[b, c[c >= 0]] |= N.MRX_LVIS_POSITIVE
            for bit, key in ((N.MRX_LVIS_NEGATIVE, "neg_category_ids"),
                             (N.MRX_LVIS_NOT_EXHAUSTIVE, "not_exhaustive_category_ids")):
                k = [self._dense(x) for x in im[key]]
                status[b, [x for x in k if x >= 0]] |= bit
        return status

    @staticmethod
    def not_exhaustive(res, status):
        """evaluate_img's last rule on a batch's downloaded flags: an unmatched detection of a
        category in its image's not_exhaustive_category_ids is ignored (a matched one still
        counts).  Updates res["ignore"] [A, T, n, R] in place where res["keep"] holds (the
        other entries of the downloaded buffer are not written on the device)."""
        nel = (status & N.MRX_LVIS_NOT_EXHAUSTIVE) != 0
        keep = res["keep"]
        cat = np.where(keep, res["cat"], 0)
        dt_nel = np.take_along_axis(nel, cat, axis=1) & keep
        res["ignore"] |= (res["match"] == -1) & dt_nel

    def _record(self, image_ids, res, gt_cats, gt_crowd, gt_area, status=None):
        """The not-exhaustive rule, then the COCO evaluator's records; status is the batch's
        `status_table`, made here from gt_cats when not given."""
        if status is None:
            status = self.status_table(image_ids, gt_cats)
        self.not_exhaustive(res, status)
        super()._record(image_ids, res, gt_cats, gt_crowd, gt_area, status)

    def _area_rng(self):
        return self.params.area_rng

    def _sync_params(self):
        self.params.img_ids = sorted(self._img_index)

    # ------------------------------------------------------------------ lvis-api's API
    def accumulate(self):
        """LVISEval's accumulate over the images of `params.img_ids` and the categories of
        `params.cat_ids`: pycocotools' per-category curves without a maxDets axis, from the
        same vectorised core as the COCO evaluators.  `eval` holds `params`, `counts` [T, R, K,
        A], `precision` [T, R, K, A] and `recall` [T, K, A] (float64, -1 where undefined)."""
        self._freeze()
        p = self.params
        img_ids = list(np.unique(p.img_ids)) if len(p.img_ids) else []
        cat_ids = [int(c) for c in p.cat_ids]
        unknown = [c for c in cat_ids if c not in self._cat_index]
        if unknown or len(set(cat_ids)) != len(cat_ids):
            raise ValueError("params.cat_ids must be distinct ids of the constructor's cat_ids")
        T, R, K, A = len(p.iou_thrs), len(p.rec_thrs), len(cat_ids), len(p.area_rng)
        precision = -np.ones((T, R, K, A))
        recall = -np.ones((T, K, A))
        for k, npig, _, score, matched, ignored in self._by_category(img_ids, cat_ids, A, T):
            for a, rc, q, _ in _curves(score, matched, ignored, npig, p.rec_thrs):
                recall[:, k, a] = rc
                precision[:, :, k, a] = q
        self.eval = {"params": p, "counts": [T, R, K, A], "precision": precision,
                     "recall": recall}

    def _summarize(self, summary_type, iou_thr=None, area_rng="all", freq_group_idx=None):
        p = self.params
        aidx = [i for i, lbl in enumerate(p.area_rng_lbl) if lbl == area_rng]
        s = self.eval["precision"] if summary_type == "ap" else self.eval["recall"]
        if iou_thr is not None:
            s = s[np.where(iou_thr == p.iou_thrs)[0]]
        if summary_type == "ap":
            if freq_group_idx is not None:
                group = [k for k, c in enumerate(p.cat_ids)
                         if self._freq[int(c)] == p.img_count_lbl[freq_group_idx]]
                s = s[:, :, group, aidx]
            else:
                s = s[:, :, :, aidx]
        else:
            s = s[:, :, aidx]
        return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])

    def summarize(self):
        """LVISEval's `results`: AP, AP50, AP75, APs, APm, APl, APr, APc, APf (the mean over the
        categories of each frequency group), AR@max_dets and ARs / ARm / ARl@max_dets, each the
        mean of the entries > -1 or -1 when there are none."""
        if not self.eval:
            raise RuntimeError("Please run accumulate() first.")
        md = self.params.max_dets
        r = self.results = OrderedDict()
        r["AP"] = self._summarize("ap")
        r["AP50"] = self._summarize("ap", iou_thr=0.50)
        r["AP75"] = self._summarize("ap", iou_thr=0.75)
        r["APs"] = self._summarize("ap", area_rng="small")
        r["APm"] = self._summarize("ap", area_rng="medium")
        r["APl"] = self._summarize("ap", area_rng="large")
        r["APr"] = self._summarize("ap", freq_group_idx=0)
        r["APc"] = self._summarize("ap", freq_group_idx=1)
        r["APf"] = self._summarize("ap", freq_group_idx=2)
        r[f"AR@{md}"] = self._summarize("ar")
        for rng in ("small", "medium", "large"):
            r[f"AR{rng[0]}@{md}"] = self._summarize("ar", area_rng=rng)

    def print_results(self):
        """`results` in lvis-api's line format."""
        template = (" {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} catIds={:>3s}] = "
                    "{:0.3f}")
        p = self.params
        for key, value in self.results.items():
            title, kind = (("Average Precision", "(AP)") if "AP" in key
                           else ("Average Recall", "(AR)"))
            if len(key) > 2 and key[2].isdigit():
                iou = "{:0.2f}".format(float(key[2:]) / 100)
            else:
                iou = "{:0.2f}:{:0.2f}".format(p.iou_thrs[0], p.iou_thrs[-1])
            group = key[2] if len(key) > 2 and key[2] in ["r", "c", "f"] else "all"
            area = key[2] if len(key) > 2 and key[2] in ["s", "m", "l"] else "all"
            print(template.format(title, kind, iou, area, p.max_dets, group, value))

    def get_results(self):
        return self.results

    def run(self):
        """evaluate(), accumulate() and summarize(), as LVISEval.run."""
        self.evaluate()
        self.accumulate()
        self.summarize()


class LVISEvalSegm(_LVISeval, COCOevalSegm):
    """lvis-api's `LVISEval(lvis_gt, LVISResults(lvis_gt, results), "segm")` (LVIS mask AP) as a
    streaming evaluator, with `COCOevalSegm`'s batch API: `add_batch` with model outputs,
    `add_results` with segm results, then `accumulate()` and `summarize()` (or `run()`) give
    LVISEval's `eval` arrays and `results`.

    `categories` and `images` are the LVIS dataset's category dicts (`id`, `frequency`) and image
    dicts (`id`, `height`, `width`, `neg_category_ids`, `not_exhaustive_category_ids`).  Per image,
    on the device (`mrx_lvis_ranks`, DESIGN.md section 3.19): only the first `max_dets` results by
    score are kept, counted over every category (LVISResults' cut); of those, a result is
    evaluated only when its category is in `cat_ids` and the image has ground truth of it or lists
    it as negative.  Then mask IoUs and matching as `COCOevalSegm`'s, with every instance
    non-crowd, and no per-(image, category) cut.  An unmatched detection of a category in the
    image's not_exhaustive_category_ids is ignored.  Ground truth is polygon lists, box lists or
    RLE dicts (`MaskBatch.from_coco`); its `area` decides its range.

    Stated differences from lvis-api: matches are recorded by position, as in `COCOevalSegm`; a
    detection's area is its mask's pixel count, where LVISResults stores w*h of the result's
    `bbox` when results carry one; NaN scores sort last, where Python's `sorted` leaves their
    order undefined; an annotation with a truthy `ignore` raises ValueError (no LVIS file carries
    the field); `eval` has no `dt_pointers`.  An image id that is not in `images`, an image dict
    without one of its keys, a category whose `frequency` is not in `img_count_lbl` and
    `max_dets` below 1 raise ValueError; `iou_thrs`, `area_rng` and `max_dets` must not change
    after the first batch."""

    _iou_type = "segm"
    _polygons = True

    def add_batch(self, items, image_ids, gt_anns, category_ids=None):
        """Evaluate model outputs against LVIS ground truth: items as for
        `api_utils.unmold_detections_batch`, one image id (of `images`) and one list of
        annotation dicts per item, `category_ids` as in `unmold_coco_results_batch`.  The kept
        masks go straight to packed planes, the annotations are rasterised on the device."""
        from . import api_utils

        api_utils.unmold_coco_eval_batch(items, image_ids, gt_anns, [self], category_ids)

    def add_results(self, results, gt_anns, image_ids):
        """Evaluate LVIS segm results -- dicts {'image_id', 'category_id', 'score',
        'segmentation': RLE dict} -- against gt_anns[b], the annotation dicts of image_ids[b].
        Every result's image must be one of image_ids; image shapes come from `images`."""
        for i in image_ids:
            if i not in self._images:
                raise ValueError(f"image {i!r} is not one of the dataset's images")
        shapes = [(int(self._images[i]["height"]), int(self._images[i]["width"]))
                  for i in image_ids]
        super().add_results(results, gt_anns, image_ids, image_shapes=shapes)


class LVISEvalBbox(_LVISeval, COCOevalBbox):
    """lvis-api's `LVISEval(lvis_gt, LVISResults(lvis_gt, results), "bbox")` (LVIS box AP) as a
    streaming evaluator: `LVISEvalSegm`'s rules and API on `COCOevalBbox`'s box IoUs (bbIou, no
    mask), every instance non-crowd; a detection's area is w*h of its box.  Annotations need
    `category_id`, `bbox` and `area`.  The stated differences are `LVISEvalSegm`'s, except the
    one on areas."""

    _iou_type = "bbox"


def ann_to_mask(ann, height, width):
    """[UPSTREAM CocoDataset.annToMask] the uint8 [height, width] mask of a COCO annotation dict,
    `decode(annToRLE(ann, height, width))`: its `segmentation` a polygon list, a box list or an
    RLE dict, rasterised or decoded on the device (`MaskBatch.from_coco`, which states what
    raises and the stated differences from pycocotools)."""
    import torch

    N.require_cuda()
    seg = ann["segmentation"] if isinstance(ann, dict) else ann
    H, W = int(height), int(width)
    gt = MaskBatch.from_coco(N.load(), torch.device("cuda", torch.cuda.current_device()),
                             [[H, W, H, W, 0, 0, H, W]], [[0]], [[seg]])
    wb = (W + 7) // 8
    o = int(gt.planes.d_packed_off[0].item())
    packed = gt.planes.d_packed[o:o + H * wb].cpu().numpy().reshape(H, wb)
    return np.unpackbits(packed, axis=1)[:, :W].copy()
