"""CPU tests of the host half of evaluate.COCOevalSegm: the vectorised accumulate against the
restated pycocotools loop (tests/cocoeval_oracle.py) on random per-detection records, the
closed form of evaluateImg's matching loop that mrx_coco_match computes, summarize()'s lines and
the ValueError cases."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest

import cocoeval_oracle as co
from matterport_maskrcnn_with_tensorflow_serving_b200 import evaluate


def _random_dataset(seed, n_img=14, n_cat=5, hw=(12, 12), max_dt=14, max_gt=6):
    """Random blob masks with crowd regions, score ties and NaN scores, and empty images."""
    rng = np.random.default_rng(seed)
    gts, dts = [], []
    for img in rng.permutation(np.arange(1, n_img + 1) * 3):
        if rng.random() < 0.15:
            continue
        for _ in range(rng.integers(0, max_gt + 1)):
            y, x = rng.integers(0, hw[0] - 2, size=2)
            m = np.zeros(hw, bool)
            m[y:y + rng.integers(1, 6), x:x + rng.integers(1, 6)] = True
            gts.append({
                "image_id": int(img), "category_id": int(rng.integers(1, n_cat + 1)), "mask": m,
                "iscrowd": int(rng.random() < 0.15),
                "area": float(rng.choice([m.sum(), 4.0, 9.0, 20.0]))})
        mine = [g for g in gts if g["image_id"] == int(img)]
        for _ in range(rng.integers(0, max_dt + 1)):
            s = float(rng.choice([0.1, 0.5, 0.5, 0.9, np.nan, rng.random()]))
            if mine and rng.random() < 0.7:      # a shifted copy of a ground-truth instance
                g = mine[rng.integers(len(mine))]
                m = np.roll(g["mask"], tuple(rng.integers(-1, 2, size=2)), axis=(0, 1))
                dts.append({"image_id": int(img), "category_id": g["category_id"], "mask": m,
                            "score": s})
                continue
            y, x = rng.integers(0, hw[0] - 2, size=2)
            m = np.zeros(hw, bool)
            m[y:y + rng.integers(0, 6), x:x + rng.integers(1, 6)] = True
            dts.append({"image_id": int(img), "category_id": int(rng.integers(1, n_cat + 2)),
                        "mask": m, "score": s})
    return gts, dts


PARAMS = [
    dict(),
    dict(maxDets=[1, 3, 5], iouThrs=np.array([0.1, 0.5, 1.0])),
    dict(areaRng=[[0, 1e10], [0, 9], [9, 20], [20, 1e10]], maxDets=[2, 4, 8]),
]


def _oracle(gts, dts, **params):
    p = co.Params()
    for k, v in params.items():
        setattr(p, k, v)
    ev = co.COCOevalOracle(gts, dts, p)
    ev.evaluate()
    ev.accumulate()
    return ev


def _product_from_oracle(ev, **params):
    """A COCOevalSegm holding the records the device would have produced for ev's images (its
    evalImgs' matches and ignore flags), in an image order other than the id order."""
    p = ev.params
    out = evaluate.COCOevalSegm(cat_ids=p.catIds, iou_thrs=p.iouThrs, max_dets=p.maxDets,
                                area_rng=p.areaRng)
    I0, A0 = len(p.imgIds), len(p.areaRng)
    order = list(reversed(p.imgIds))
    for pos, img in enumerate(order):
        out._img_index[img] = pos
    for c in p.catIds:
        out._dense(c)
    img, cat, rank, score, tp, ig = [], [], [], [], [], []
    for k, c in enumerate(p.catIds):
        for i, im in enumerate(p.imgIds):
            es = [ev.evalImgs[k * A0 * I0 + a * I0 + i] for a in range(A0)]
            if es[0] is None:
                continue
            D = len(es[0]["dtScores"])
            img += [out._img_index[im]] * D
            cat += [out._cat_index[c]] * D
            rank += list(range(D))
            score += es[0]["dtScores"]
            tp.append(np.stack([e["dtMatches"].T > -1 for e in es], axis=1))
            ig.append(np.stack([e["dtIgnore"].T.astype(bool) for e in es], axis=1))
    T = len(p.iouThrs)
    out._dets.append((np.array(img, np.int64), np.array(cat, np.int32), np.array(rank, np.int32),
                      np.array(score, np.float64), np.concatenate(tp + [np.zeros((0, A0, T), bool)]),
                      np.concatenate(ig + [np.zeros((0, A0, T), bool)])))
    rngs = np.asarray(p.areaRng, np.float64)
    g = [x for x in ev.gts_in if x["category_id"] in p.catIds]
    nonig = np.array([[not x["iscrowd"] and lo <= x["area"] <= hi for lo, hi in rngs] for x in g],
                     bool).reshape(-1, A0)
    out._gts.append((np.array([out._img_index[x["image_id"]] for x in g], np.int64),
                     np.array([out._cat_index[x["category_id"]] for x in g], np.int32), nonig))
    out.params.imgIds = list(p.imgIds)
    out.params.recThrs = p.recThrs
    return out


def _same(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("params", range(len(PARAMS)))
def test_accumulate_equals_the_loop(seed, params):
    gts, dts = _random_dataset(seed)
    ev = _oracle(gts, dts, **PARAMS[params])
    got = _product_from_oracle(ev)
    got.accumulate()
    for name in ("precision", "recall", "scores"):
        _same(got.eval[name], ev.eval[name])
    assert got.eval["counts"] == ev.eval["counts"]
    assert (ev.eval["precision"] > 0).any()
    with redirect_stdout(io.StringIO()) as a:
        ev.summarize()
    with redirect_stdout(io.StringIO()) as b:
        got.summarize()
    assert a.getvalue() == b.getvalue()
    assert np.array_equal(ev.stats, got.stats)


def test_accumulate_image_and_category_subsets():
    gts, dts = _random_dataset(7)
    ev = _oracle(gts, dts)
    got = _product_from_oracle(ev)
    keep_imgs, keep_cats = ev.params.imgIds[::2], ev.params.catIds[1:]
    sub = _oracle(gts, dts, imgIds=list(keep_imgs), catIds=list(keep_cats))
    got.params.imgIds, got.params.catIds = list(keep_imgs), list(keep_cats)
    got.accumulate()
    for name in ("precision", "recall", "scores"):
        _same(got.eval[name], sub.eval[name])


def closed_form(ious, crowd, gt_ig, thresholds):
    """What mrx_coco_match computes for one (image, category, area range): per threshold and
    detection (in score order), the gt index (caller's order) or -1 and the ignore flag."""
    T, (D, G) = len(thresholds), ious.shape
    dtm = -np.ones((T, D), np.int64)
    dtig = np.zeros((T, D), bool)
    for t, thr in enumerate(thresholds):
        matched = np.zeros(G, bool)
        for d in range(D):
            cand = (~matched | crowd) & (ious[d] >= min(thr, 1 - 1e-10))
            for group in (~gt_ig, gt_ig):
                c = np.nonzero(cand & group)[0]
                if c.size:
                    best = ious[d, c].max()
                    j = c[ious[d, c] == best][-1]
                    dtm[t, d], dtig[t, d] = j, gt_ig[j]
                    matched[j] = True
                    break
    return dtm, dtig


@pytest.mark.parametrize("seed", [4, 5])
def test_closed_form_matching_equals_the_loop(seed):
    gts, dts = _random_dataset(seed, hw=(8, 8), max_dt=20, max_gt=10)
    ev = _oracle(gts, dts, iouThrs=np.array([0.0, 0.2, 0.5, 1.0]))
    p = ev.params
    checked = 0
    for k, c in enumerate(p.catIds):
        for a, rng in enumerate(p.areaRng):
            for i, im in enumerate(p.imgIds):
                e = ev.evalImgs[k * len(p.areaRng) * len(p.imgIds) + a * len(p.imgIds) + i]
                g = ev._gts[im, c]
                if e is None or not len(ev.ious[im, c]):
                    continue
                crowd = np.array([x["iscrowd"] for x in g], bool)
                area = np.array([x["area"] for x in g])
                ig = crowd | (area < rng[0]) | (area > rng[1])
                dtm, dtig = closed_form(ev.ious[im, c], crowd, ig, p.iouThrs)
                pos = {x["id"]: j for j, x in enumerate(g)}
                want = np.vectorize(lambda v: pos.get(v, -1))(e["dtMatchIds"])
                assert np.array_equal(dtm, want)
                d_area = np.array([x["mask"].sum() for x in ev._dts[im, c]])
                d_area = d_area[np.argsort([-x["score"] for x in ev._dts[im, c]],
                                           kind="mergesort")][:dtm.shape[1]]
                dtig |= (dtm == -1) & ((d_area < rng[0]) | (d_area > rng[1]))[None]
                assert np.array_equal(dtig, e["dtIgnore"])
                checked += 1
    assert checked > 20


def test_summarize_prints_pycocotools_lines():
    m = np.zeros((20, 20), bool)
    m[5:15, 5:15] = True
    ev = _oracle([{"image_id": 1, "category_id": 1, "mask": m, "iscrowd": 0, "area": 100.0}],
                 [{"image_id": 1, "category_id": 1, "mask": m, "score": 0.9}])
    got = _product_from_oracle(ev)
    got.accumulate()
    with redirect_stdout(io.StringIO()) as out:
        got.summarize()
    assert out.getvalue() == """\
 Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = 1.000
 Average Precision  (AP) @[ IoU=0.50      | area=   all | maxDets=100 ] = 1.000
 Average Precision  (AP) @[ IoU=0.75      | area=   all | maxDets=100 ] = 1.000
 Average Precision  (AP) @[ IoU=0.50:0.95 | area= small | maxDets=100 ] = 1.000
 Average Precision  (AP) @[ IoU=0.50:0.95 | area=medium | maxDets=100 ] = -1.000
 Average Precision  (AP) @[ IoU=0.50:0.95 | area= large | maxDets=100 ] = -1.000
 Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets=  1 ] = 1.000
 Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets= 10 ] = 1.000
 Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = 1.000
 Average Recall     (AR) @[ IoU=0.50:0.95 | area= small | maxDets=100 ] = 1.000
 Average Recall     (AR) @[ IoU=0.50:0.95 | area=medium | maxDets=100 ] = -1.000
 Average Recall     (AR) @[ IoU=0.50:0.95 | area= large | maxDets=100 ] = -1.000
"""
    assert got.eval["params"] is got.params and got.eval["counts"] == [10, 101, 1, 4, 3]


def test_default_params_are_pycocotools():
    p, q = evaluate.COCOevalSegm().params, co.Params()
    for name in ("iouThrs", "recThrs", "maxDets", "areaRng", "areaRngLbl", "useCats"):
        assert np.array_equal(getattr(p, name), getattr(q, name)), name


RLE = {"size": [4, 6], "counts": b"0j0"}
ITEM = (np.zeros((2, 6), np.float32), np.zeros((2, 28, 28, 3), np.float32), (4, 6, 3),
        (16, 16, 3), (0, 0, 11, 16))


@pytest.mark.parametrize("call,msg", [
    (lambda e: e.add_batch([ITEM], [1], [[{"category_id": 1, "segmentation": [[0, 0, 1, 1, 2, 0]],
                                           "id": 77}]]), r"image 1, annotation 0 \(id 77\): polygon"),
    (lambda e: e.add_batch([ITEM], [1], [[{"category_id": 1,
                                           "segmentation": {"size": [5, 6], "counts": b"0m0"}}]]),
     r"RLE size \[5, 6\] is not the image's \[4, 6\]"),
    (lambda e: e.add_batch([ITEM, ITEM], [3, 3], [[], []]), "image 3 was already added"),
    (lambda e: e.add_batch([ITEM], [1, 2], [[], []]), "1 items but 2 image ids"),
    (lambda e: e.add_batch([ITEM], [1], []), "0 ground-truth annotation lists for 1 images"),
    (lambda e: e.add_results([], [[], []], [1]), "2 annotation lists but 1 image ids"),
    (lambda e: e.add_results([{"image_id": 9, "category_id": 1, "score": 1.0,
                               "segmentation": RLE}], [[]], [1]), "result 0: image 9 is not one"),
    (lambda e: e.add_results([{"image_id": 1, "category_id": 1, "score": 1.0,
                               "segmentation": RLE}],
                             [[{"category_id": 1, "segmentation": {"size": [4, 5], "counts": b"0"}}]],
                             [1]), r"image 1: RLE sizes .* differ"),
    (lambda e: e.add_results([{"image_id": 1, "category_id": 1, "score": 1.0,
                               "segmentation": [[0, 0, 1, 1]]}], [[]], [1]),
     "result 0: segmentation must be an RLE dict"),
])
def test_value_errors(call, msg):
    with pytest.raises(ValueError, match=msg):
        call(evaluate.COCOevalSegm())


def test_image_added_in_an_earlier_batch_is_refused():
    ev = evaluate.COCOevalSegm()
    ev._img_index[5] = 0
    with pytest.raises(ValueError, match="image 5 was already added"):
        ev.add_results([], [[]], [5])


def test_params_outside_the_kernels_limits():
    with pytest.raises(ValueError, match="IoU thresholds"):
        evaluate.COCOevalSegm(iou_thrs=np.linspace(0, 1, 65))
    with pytest.raises(ValueError, match="area ranges"):
        evaluate.COCOevalSegm(area_rng=[[0, 1]] * 17, area_rng_lbl=list("abcdefghijklmnopq"))
    ev = evaluate.COCOevalSegm()
    ev._freeze()
    ev.params.iouThrs = np.array([0.5])
    with pytest.raises(ValueError, match="changed after the first batch"):
        ev.accumulate()
