"""COCO mask evaluation on the device (mrx_coco_ranks / _ious / _match and evaluate.COCOevalSegm):
everything must equal the restated pycocotools COCOeval (tests/cocoeval_oracle.py) run on the
masks unmold_detections_batch returns -- IoUs bit for bit, match and ignore flags for every
(area range, threshold), and the accumulated arrays and stats exactly."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest

import cocoeval_oracle as co
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate, synth

from helpers import item_of

pytestmark = pytest.mark.gpu


def rle_of(m):
    """Uncompressed COCO RLE of a bool [H, W] mask (column-major runs starting with zeros)."""
    f = np.asarray(m, bool).ravel(order="F")
    ends = np.concatenate([np.flatnonzero(f[1:] != f[:-1]) + 1, [f.size]])
    runs = np.diff(np.concatenate([[0], ends]))
    if f.size and f[0]:
        runs = np.concatenate([[0], runs])
    return {"size": list(m.shape), "counts": [int(v) for v in runs]}


class Capture(evaluate.COCOevalSegm):
    """Keeps every batch's device results for the per-pair checks."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.batches = []

    def _record(self, image_ids, res, *rest):
        self.batches.append((list(image_ids), res))
        super()._record(image_ids, res, *rest)


def make_batch(seed, shapes, n, R, classes, ties=True):
    """items, ground-truth annotation lists and the bool masks of both sides for one batch."""
    rng = np.random.default_rng(seed)
    ims = [synth.make_image(rng, hw, n, num_classes=classes, max_instances=R,
                            **({} if min(hw) > 64 else dict(min_box=1, max_box_frac=1.0)))
           for hw in shapes]
    for im in ims:
        if ties:       # equal scores within an image and across images
            im.detections[:im.n_valid, 5] = np.round(im.detections[:im.n_valid, 5], 1)
    items = [item_of(im, np.float32) for im in ims]
    jit = [synth.jitter_coco_ground_truth(im, rng, crowd_frac=0.1, max_shift=3,
                                          class_flip_frac=0.2) for im in ims]
    gt_out = api_utils.unmold_detections_batch([item_of(j, np.float32) for j, _, _ in jit])
    anns, gt_masks = [], []
    for (_, crowd, area), (_, cls, _, masks) in zip(jit, gt_out):
        a, ms = [], []
        for k in range(cls.shape[0]):
            ann = {"category_id": int(cls[k]), "segmentation": rle_of(masks[:, :, k]),
                   "iscrowd": int(crowd[k]), "area": float(area[k]), "id": k + 1}
            if k % 7 == 3:
                del ann["area"]                 # the mask's pixel count stands in
            a.append(ann)
            ms.append(masks[:, :, k])
        H, W = masks.shape[:2]
        a.append({"category_id": int(cls[0]) if cls.size else 1, "iscrowd": 0, "area": 50.0,
                  "segmentation": rle_of(np.zeros((H, W), bool))})     # an empty mask
        ms.append(np.zeros((H, W), bool))
        anns.append(a)
        gt_masks.append(ms)
    preds = api_utils.unmold_detections_batch(items)
    return items, anns, gt_masks, preds


def oracle_inputs(batches, category_ids=None):
    """(gts, dts, gmap, dmap) for the oracle: gmap[gid] = (image id, j), dmap[did] = (image id,
    kept index i)."""
    gts, dts, gmap, dmap = [], [], {}, {}
    for ids, items, anns, gt_masks, preds in batches:
        for img, a, ms, (_, cls, scores, masks) in zip(ids, anns, gt_masks, preds):
            for j, (ann, m) in enumerate(zip(a, ms)):
                gmap[len(gts)] = (img, j)
                gts.append({"image_id": img, "category_id": ann["category_id"], "mask": m,
                            "iscrowd": ann["iscrowd"],
                            "area": ann.get("area", float(m.sum()))})
            for i in range(cls.shape[0]):
                dmap[len(dts)] = (img, i)
                c = int(cls[i])
                dts.append({"image_id": img, "mask": masks[:, :, i], "score": float(scores[i]),
                            "category_id": c if category_ids is None else int(category_ids[c])})
    return gts, dts, gmap, dmap


def run_oracle(gts, dts, **params):
    p = co.Params()
    for k, v in params.items():
        setattr(p, k, v)
    ev = co.COCOevalOracle(gts, dts, p)
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
    ([7], [(800, 1333)], 60, 64, 4),
]


@pytest.mark.parametrize("params", [
    dict(),
    dict(iouThrs=np.array([0.3, 0.5, 0.75, 1.0]), maxDets=[1, 5, 20]),
    dict(areaRng=[[0, 1e10], [0, 100], [100, 2000], [2000, 1e10], [1024, 9216]],
         areaRngLbl=["all", "small", "medium", "large", "mid"], maxDets=[2, 10, 20]),
])
def test_stream_equals_oracle(cuda_device, params):
    batches = []
    for s, (ids, shapes, n, R, classes) in enumerate(STREAM):
        batches.append((ids,) + make_batch(200 + s, shapes, n, R, classes))
    kw = {"iou_thrs": params.get("iouThrs"), "max_dets": params.get("maxDets", (1, 10, 100)),
          "area_rng": params.get("areaRng"), "area_rng_lbl": params.get("areaRngLbl")}
    got = Capture(**kw)
    for ids, items, anns, _, _ in batches:
        api_utils.unmold_coco_eval_batch(items, ids, anns, got)
    got.evaluate()
    got.accumulate()
    gts, dts, gmap, dmap = oracle_inputs(batches)
    ev = run_oracle(gts, dts, **params)
    assert got.params.imgIds == ev.params.imgIds and got.params.catIds == ev.params.catIds
    n_iou, n_flags = check_pairs(ev, got, gmap, dmap)
    assert n_iou > 500 and n_flags > 500
    same_eval(got, ev)
    assert (ev.eval["precision"] > 0).any()
    if "maxDets" in params:        # more than maxDets[-1] predictions in some (image, category)
        assert max(len(v) for v in ev._dts.values()) > params["maxDets"][-1]


def test_full_size_crowds_and_category_map(cuda_device):
    """A configs[1] image (1024 x 1024, 100 predictions against 100 jittered instances) and an
    800 x 1333 one, class ids mapped to other category ids."""
    rng = np.random.default_rng(301)
    ims = [synth.make_image(rng, (1024, 1024), 100, num_classes=81, max_instances=100,
                            mold=((1024, 1024, 3), (0, 0, 1024, 1024)))]
    ims.append(synth.make_image(rng, (800, 1333), 100, num_classes=81, max_instances=100))
    items = [item_of(im, np.float32) for im in ims]
    jit = [synth.jitter_coco_ground_truth(im, rng, crowd_frac=0.1) for im in ims]
    gt_out = api_utils.unmold_detections_batch([item_of(j, np.float32) for j, _, _ in jit])
    anns, gt_masks = [], []
    for (_, crowd, area), (_, cls, _, masks) in zip(jit, gt_out):
        anns.append([{"category_id": 1000 + int(cls[k]), "iscrowd": int(crowd[k]),
                      "area": float(area[k]), "segmentation": rle_of(masks[:, :, k])}
                     for k in range(cls.shape[0])])
        gt_masks.append([masks[:, :, k] for k in range(cls.shape[0])])
    cmap = {c: 1000 + c for c in range(81)}
    preds = api_utils.unmold_detections_batch(items)
    got = Capture()
    api_utils.unmold_coco_eval_batch(items, [2, 1], anns, got, category_ids=cmap)
    got.accumulate()
    batches = [([2, 1], items, anns, gt_masks, preds)]
    gts, dts, gmap, dmap = oracle_inputs(batches, cmap)
    ev = run_oracle(gts, dts)
    n_iou, _ = check_pairs(ev, got, gmap, dmap)
    assert n_iou > 50 and any(g["iscrowd"] for g in gts)
    same_eval(got, ev)


def test_add_results_equals_add_batch(cuda_device):
    a, b = evaluate.COCOevalSegm(max_dets=(1, 5, 20)), evaluate.COCOevalSegm(max_dets=(1, 5, 20))
    for s, (ids, shapes, n, R, classes) in enumerate(STREAM):
        items, anns, _, _ = make_batch(400 + s, shapes, n, R, classes)
        cmap = [10 * c + 3 for c in range(classes)]
        for a_ in anns:
            for ann in a_:
                ann["category_id"] = cmap[ann["category_id"]]
        a.add_batch(items, ids, anns, category_ids=cmap)
        results = api_utils.unmold_coco_results_batch(items, ids, category_ids=cmap)
        if s == 1:      # the strings as JSON holds them
            for r in results:
                r["segmentation"] = dict(r["segmentation"],
                                         counts=r["segmentation"]["counts"].decode("ascii"))
        b.add_results(results, anns, ids)
    a.accumulate()
    b.accumulate()
    for name in ("precision", "recall", "scores"):
        assert np.array_equal(a.eval[name].view(np.uint64), b.eval[name].view(np.uint64)), name
    assert (a.eval["precision"] > 0).any()
