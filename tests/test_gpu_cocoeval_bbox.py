"""COCO box evaluation on the device (mrx_coco_box_ious / mrx_coco_match_f64area and
evaluate.COCOevalBbox): everything must equal the restated pycocotools COCOeval for "bbox"
(tests/bbox_cocoeval_oracle.py) -- IoUs bit for bit, match and ignore flags for every (area range,
threshold), and the accumulated arrays and stats exactly -- with no mask expanded, and one unmold
must feed a segm and a bbox evaluator as two separate add_batch calls would."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

import bbox_cocoeval_oracle as bo
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate, synth
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import (UnmoldEngine,
                                                                     coco_box_evaluate_batch)

from helpers import item_of
from test_host_cocoeval_bbox import FUSED_D, FUSED_G, fused_iou

pytestmark = pytest.mark.gpu


class Capture(evaluate.COCOevalBbox):
    """Keeps every batch's device results for the per-pair checks."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.batches = []

    def _record(self, image_ids, res, *rest):
        self.batches.append((list(image_ids), res))
        super()._record(image_ids, res, *rest)


def float_boxes(rng, yxyx):
    """COCO-file ground-truth boxes [x, y, w, h] from int (y1, x1, y2, x2) mask extents: sub-pixel
    jitter, rounded to 2 decimals as COCO files store them, a few zero or negative widths and
    heights, and a few exact duplicates of another box (IoU ties)."""
    b = np.asarray(yxyx, np.float64).reshape(-1, 4)
    n = b.shape[0]
    xywh = np.stack([b[:, 1], b[:, 0], b[:, 3] - b[:, 1], b[:, 2] - b[:, 0]], axis=1)
    xywh = np.round(xywh + rng.uniform(-0.5, 0.5, size=(n, 4)), 2)
    for k in range(n):
        r = rng.random()
        if r < 0.04:
            xywh[k, 2 + (k & 1)] = 0.0
        elif r < 0.08:
            xywh[k, 2 + (k & 1)] = -np.round(rng.uniform(0.01, 5), 2)
        elif r < 0.14 and k:
            xywh[k] = xywh[rng.integers(k)]
    return xywh


def make_batch(seed, shapes, n, R, classes, cmap):
    """items and ground-truth annotations (bbox, area, iscrowd, a compressed-RLE segmentation)
    for one batch; category ids through cmap."""
    rng = np.random.default_rng(seed)
    ims = [synth.make_image(rng, hw, n, num_classes=classes, max_instances=R,
                            **({} if min(hw) > 64 else dict(min_box=1, max_box_frac=1.0)))
           for hw in shapes]
    for im in ims:       # equal scores within an image and across images
        im.detections[:im.n_valid, 5] = np.round(im.detections[:im.n_valid, 5], 1)
    items = [item_of(im, np.float32) for im in ims]
    jit = [synth.jitter_coco_ground_truth(im, rng, crowd_frac=0.1, max_shift=3,
                                          class_flip_frac=0.2) for im in ims]
    gt_out = api_utils.unmold_detections_rle_batch([item_of(j, np.float32) for j, _, _ in jit],
                                                   compressed=True)
    anns = []
    for (_, crowd, area), (boxes, cls, _, rles) in zip(jit, gt_out):
        bb = float_boxes(rng, boxes)
        anns.append([{"category_id": cmap[int(cls[k])], "bbox": [float(v) for v in bb[k]],
                      "iscrowd": int(crowd[k]), "area": float(area[k]), "id": k + 1,
                      "segmentation": rles[k]} for k in range(cls.shape[0])])
    return items, anns


def oracle_inputs(batches, cmap):
    """(gts, dts, gmap, dmap) for the oracle from the kept boxes unmold_detections returns:
    gmap[gid] = (image id, j), dmap[did] = (image id, kept index i)."""
    gts, dts, gmap, dmap = [], [], {}, {}
    for ids, items, anns in batches:
        preds = api_utils.unmold_detections_packed_batch(items)
        for img, a, (boxes, cls, scores, _) in zip(ids, anns, preds):
            for j, ann in enumerate(a):
                gmap[len(gts)] = (img, j)
                gts.append({"image_id": img, "category_id": ann["category_id"],
                            "bbox": ann["bbox"], "iscrowd": ann["iscrowd"], "area": ann["area"]})
            for i in range(cls.shape[0]):
                dmap[len(dts)] = (img, i)
                y1, x1, y2, x2 = (int(v) for v in boxes[i])
                dts.append({"image_id": img, "category_id": cmap[int(cls[i])],
                            "bbox": [x1, y1, x2 - x1, y2 - y1], "score": float(scores[i])})
    return gts, dts, gmap, dmap


def run_oracle(gts, dts, **params):
    p = bo.Params()
    for k, v in params.items():
        setattr(p, k, v)
    ev = bo.COCOevalBboxOracle(gts, dts, p)
    ev.evaluate()
    ev.accumulate()
    with redirect_stdout(io.StringIO()) as out:
        ev.summarize()
    ev.printed = out.getvalue()
    return ev


def check_pairs(ev, got, gmap, dmap):
    """Device IoUs, ranks, match and ignore flags against the oracle's computeIoU / evaluateImg."""
    p = ev.params
    where = {}
    for ids, res in got.batches:
        for b, img in enumerate(ids):
            where[img] = (b, res)
    inv_cat = {d: c for c, d in got._cat_index.items()}
    n_iou = n_flags = 0
    for (img, cat), ious in ev.ious.items():
        if not len(ious):
            continue
        b, res = where[img]
        d_iou = res["d_iou"][b].cpu().numpy()
        order = np.argsort([-d["score"] for d in ev._dts[img, cat]], kind="mergesort")
        dts = [ev._dts[img, cat][o] for o in order][:p.maxDets[-1]]
        for di, d in enumerate(dts):
            i = dmap[d["id"]][1]
            assert res["keep"][b, i] and res["rank"][b, i] == di
            assert inv_cat[res["cat"][b, i]] == cat
            assert res["area"][b, i] == d["area"]
            for gi, g in enumerate(ev._gts[img, cat]):
                j = gmap[g["id"]][1]
                assert d_iou[i, j].view(np.uint64) == np.float64(ious[di, gi]).view(np.uint64), \
                    (img, cat, i, j, d_iou[i, j], ious[di, gi])
                n_iou += 1
    nI, nA = len(p.imgIds), len(p.areaRng)
    for k, cat in enumerate(p.catIds):
        for a in range(nA):
            for ii, img in enumerate(p.imgIds):
                e = ev.evalImgs[k * nA * nI + a * nI + ii]
                if e is None:
                    continue
                b, res = where[img]
                for di, did in enumerate(e["dtIds"]):
                    i = dmap[did][1]
                    want = [gmap[g][1] if g > -1 else -1 for g in e["dtMatchIds"][:, di]]
                    assert np.array_equal(res["match"][a, :, b, i], want), (img, cat, a, i)
                    assert np.array_equal(res["ignore"][a, :, b, i], e["dtIgnore"][:, di] != 0)
                    n_flags += 1
    return n_iou, n_flags


def same_eval(got, ev):
    for name in ("precision", "recall", "scores"):
        a, b = got.eval[name], ev.eval[name]
        assert a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64)), name
    with redirect_stdout(io.StringIO()) as out:
        got.summarize()
    assert out.getvalue() == ev.printed
    assert np.array_equal(got.stats, ev.stats)


STREAM = [  # (image ids, shapes, n, R, classes)
    ([30, 10], [(17, 9), (75, 333)], 12, 16, 3),
    ([20, 5, 40], [(96, 128), (33, 100), (64, 64)], 40, 48, 3),
    ([7], [(800, 1333)], 60, 64, 3),
]
CMAP = [10 * c + 3 for c in range(3)]


def stream_batches(seed):
    return [(ids,) + make_batch(seed + s, shapes, n, R, classes, CMAP)
            for s, (ids, shapes, n, R, classes) in enumerate(STREAM)]


# ----------------------------------------------------------------------------- IoUs
def _random_case(rng, n_img=3, R1=40, R2=50):
    cats = 3
    M = rng.integers(1, R2 + 1, size=n_img)
    M[1] = R2
    Nn = rng.integers(1, R1 + 1, size=n_img)
    Nn[0] = R1
    gt_yxyx = []
    for b in range(n_img):
        y1, x1 = rng.integers(0, 500, size=(2, R2))
        gt_yxyx.append(np.stack([y1, x1, y1 + rng.integers(1, 300, R2), x1 + rng.integers(1, 300, R2)],
                                axis=1))
    gt_boxes = np.stack([float_boxes(rng, g) for g in gt_yxyx])
    gt_cat = rng.integers(0, cats, size=(n_img, R2)).astype(np.int32)
    gt_crowd = (rng.random((n_img, R2)) < 0.2).astype(np.uint8)
    # predictions: shifted copies of ground-truth extents, so most pairs overlap
    src = rng.integers(0, R2, size=(n_img, R1))
    pred_yxyx = np.stack([g[s] for g, s in zip(gt_yxyx, src)]) + rng.integers(-20, 21, (n_img, R1, 4))
    pred_yxyx[..., 2:] = np.maximum(pred_yxyx[..., 2:], pred_yxyx[..., :2] + 1)
    pred_cat = np.stack([c[s] for c, s in zip(gt_cat, src)])
    pred_cat[rng.random((n_img, R1)) < 0.2] = rng.integers(0, cats)
    scores = np.round(rng.random((n_img, R1)), 1)
    # the pair whose fused and unfused forms round apart
    gt_boxes[0, 0], gt_cat[0, 0], gt_crowd[0, 0], pred_cat[0, 0] = FUSED_G, 0, 0, 0
    return dict(M=M.astype(np.int32), N=Nn.astype(np.int32), gt_boxes=gt_boxes, gt_cat=gt_cat,
                gt_crowd=gt_crowd, pred_yxyx=pred_yxyx.astype(np.int32),
                pred_cat=pred_cat.astype(np.int32), scores=scores)


@pytest.mark.parametrize("form", ["yxyx_int32_device", "xywh_float64_host"])
def test_box_ious_equal_bbiou(cuda_device, form):
    rng = np.random.default_rng(17 if form[0] == "y" else 18)
    c = _random_case(rng)
    n, R1, R2 = c["pred_yxyx"].shape[0], c["pred_yxyx"].shape[1], c["gt_cat"].shape[1]
    b_ = c["pred_yxyx"]
    xywh = np.stack([b_[..., 1], b_[..., 0], b_[..., 3] - b_[..., 1], b_[..., 2] - b_[..., 0]],
                    axis=-1).astype(np.float64)
    if form[0] == "y":
        pred_boxes = torch.from_numpy(c["pred_yxyx"]).cuda()
        pred_cls = torch.from_numpy(c["pred_cat"]).cuda()
        scores = torch.from_numpy(c["scores"].astype(np.float32)).cuda()
    else:
        xywh = float_boxes(rng, c["pred_yxyx"].reshape(-1, 4)).reshape(n, R1, 4)
        xywh[0, 0] = FUSED_D
        pred_boxes, pred_cls, scores = xywh, c["pred_cat"], c["scores"]
    res = coco_box_evaluate_batch(N.load(), pred_boxes, c["N"], pred_cls, scores, c["M"],
                                  c["gt_cat"], c["gt_boxes"], c["gt_crowd"],
                                  np.full((n, R2), 100.0), np.arange(3, dtype=np.int32),
                                  evaluate.Params())
    iou = res["d_iou"].cpu().numpy()
    pairs = crowd_pairs = zero = 0
    for b in range(n):
        for i in range(c["N"][b]):
            assert res["keep"][b, i]
            D = xywh[b, i]
            assert res["area"][b, i] == D[2] * D[3]
            for j in range(c["M"][b]):
                if c["gt_cat"][b, j] != c["pred_cat"][b, i]:
                    continue
                want = bo.bb_iou([D], [c["gt_boxes"][b, j]], [c["gt_crowd"][b, j]])[0, 0]
                assert iou[b, i, j].view(np.uint64) == np.float64(want).view(np.uint64), \
                    (b, i, j, iou[b, i, j], want)
                pairs += 1
                crowd_pairs += int(c["gt_crowd"][b, j])
                zero += want == 0
    assert pairs > 800 and crowd_pairs > 50 and 100 < zero < pairs - 100
    if form[0] == "x":
        assert iou[0, 0, 0] == bo.bb_iou([FUSED_D], [FUSED_G], [0])[0, 0]
        assert iou[0, 0, 0] != fused_iou(FUSED_D, FUSED_G)


# ----------------------------------------------------------------------------- evaluator
@pytest.mark.parametrize("params", [
    dict(),
    dict(iouThrs=np.array([0.3, 0.5, 0.75, 1.0]), maxDets=[1, 5, 20]),
    dict(areaRng=[[0, 1e10], [0, 100], [100, 2000], [2000, 1e10], [1024, 9216]],
         areaRngLbl=["all", "small", "medium", "large", "mid"], maxDets=[2, 10, 20]),
])
def test_add_batch_equals_oracle(cuda_device, params):
    batches = stream_batches(500)
    kw = {"iou_thrs": params.get("iouThrs"), "max_dets": params.get("maxDets", (1, 10, 100)),
          "area_rng": params.get("areaRng"), "area_rng_lbl": params.get("areaRngLbl")}
    got = Capture(**kw)
    for ids, items, anns in batches:
        got.add_batch(items, ids, anns, category_ids=CMAP)
    got.evaluate()
    got.accumulate()
    gts, dts, gmap, dmap = oracle_inputs(batches, CMAP)
    ev = run_oracle(gts, dts, **params)
    assert got.params.imgIds == ev.params.imgIds and got.params.catIds == ev.params.catIds
    n_iou, n_flags = check_pairs(ev, got, gmap, dmap)
    assert n_iou > 500 and n_flags > 500
    same_eval(got, ev)
    assert (ev.eval["precision"] > 0).any()
    if "maxDets" in params:        # more than maxDets[-1] predictions in some (image, category)
        assert max(len(v) for v in ev._dts.values()) > params["maxDets"][-1]


def test_add_results_equals_oracle(cuda_device):
    batches = stream_batches(600)
    got = Capture(max_dets=(1, 5, 20))
    for ids, items, anns in batches:
        got.add_results(api_utils.unmold_coco_results_batch(items, ids, category_ids=CMAP), anns,
                        ids)
    got.accumulate()
    gts, dts, gmap, dmap = oracle_inputs(batches, CMAP)
    ev = run_oracle(gts, dts, maxDets=[1, 5, 20])
    n_iou, n_flags = check_pairs(ev, got, gmap, dmap)
    assert n_iou > 500 and n_flags > 500
    same_eval(got, ev)


def test_add_batch_expands_no_mask(cuda_device, monkeypatch):
    batches = stream_batches(700)[:2]
    calls = []

    def refuse(name):
        def f(*a, **kw):
            raise AssertionError(f"{name} called by a bbox evaluation")
        return f

    for name in ("enqueue_expand", "enqueue_expand_packed", "enqueue_packed", "pack_masks",
                 "enqueue_rle", "ground_truth_rle", "ground_truth_coco"):
        monkeypatch.setattr(UnmoldEngine, name, refuse(name))
    prepare = UnmoldEngine.enqueue
    monkeypatch.setattr(UnmoldEngine, "enqueue",
                        lambda self, *a, **kw: (calls.append(kw.get("expand", True)),
                                                prepare(self, *a, **kw))[1])
    got = evaluate.COCOevalBbox()
    for ids, items, anns in batches:
        for a in anns:
            for k, ann in enumerate(a):      # no segmentation is read: any value or none at all
                if k % 3 == 0:
                    del ann["segmentation"]
                elif k % 3 == 1:
                    ann["segmentation"] = [[0.0, 0.0, 5.0, 0.0, 5.0, 5.0]]
        got.add_batch(items, ids, anns, category_ids=CMAP)
    assert calls == [False, False]
    got.accumulate()
    assert (got.eval["precision"] > 0).any()


def test_one_unmold_for_both_evaluators(cuda_device, monkeypatch):
    batches = stream_batches(800)
    kw = dict(max_dets=(1, 5, 20))
    both = [evaluate.COCOevalSegm(**kw), evaluate.COCOevalBbox(**kw)]
    apart = [evaluate.COCOevalSegm(**kw), evaluate.COCOevalBbox(**kw)]
    for ids, items, anns in batches:
        for e in apart:
            e.add_batch(items, ids, anns, category_ids=CMAP)
    prepares = []
    prepare = UnmoldEngine.enqueue
    monkeypatch.setattr(UnmoldEngine, "enqueue",
                        lambda self, *a, **kw: (prepares.append(1), prepare(self, *a, **kw))[1])
    for ids, items, anns in batches:
        api_utils.unmold_coco_eval_batch(items, ids, anns, both, category_ids=CMAP)
    assert len(prepares) == len(batches)
    for a, b in zip(both, apart):
        for e in (a, b):
            e.accumulate()
            with redirect_stdout(io.StringIO()):
                e.summarize()
        for name in ("precision", "recall", "scores"):
            assert np.array_equal(a.eval[name].view(np.uint64), b.eval[name].view(np.uint64))
        assert np.array_equal(a.stats.view(np.uint64), b.stats.view(np.uint64))
        assert (a.eval["precision"] > 0).any()
    assert not np.array_equal(both[0].stats, both[1].stats)
