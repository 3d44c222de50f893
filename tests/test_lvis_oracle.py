"""Known answers of the restated LVISEval (tests/lvis_oracle.py), one per rule, each of which flips
a result, and its cross-check against the restated COCOeval where the two must agree."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest

import cocoeval_oracle as co
import lvis_oracle as lo

ONE = 1 / (1 + np.spacing(1))     # tp / (fp + tp + eps) of a perfect curve
CATS = [{"id": 1, "frequency": "r"}, {"id": 2, "frequency": "f"}, {"id": 3, "frequency": "f"}]


def image(i, neg=(), nel=()):
    return {"id": i, "height": 200, "width": 200, "neg_category_ids": list(neg),
            "not_exhaustive_category_ids": list(nel)}


def gt(img, cat, bbox, **kw):
    return dict({"image_id": img, "category_id": cat, "bbox": list(bbox),
                 "area": float(bbox[2] * bbox[3])}, **kw)


def dt(img, cat, bbox, score):
    return {"image_id": img, "category_id": cat, "bbox": list(bbox), "score": score}


def run(gts, dts, images, max_dets=300, cats=CATS):
    p = lo.Params("bbox")
    p.max_dets = max_dets
    ev = lo.LVISEvalOracle(gts, dts, images, cats, "bbox", p)
    ev.run()
    return ev


BOX = (0, 0, 10, 10)
FAR = (100, 100, 10, 10)


def test_the_301st_detection_is_cut_and_its_ground_truth_becomes_a_miss():
    gts = [gt(1, 1, BOX), gt(1, 2, FAR)]
    dts = [dt(1, 2, (150, 150, 5, 5), 0.9) for _ in range(300)] + [dt(1, 1, BOX, 0.5)]
    cut = run(gts, dts, [image(1)])
    assert np.all(cut.eval["recall"][:, 0, 0] == 0)
    assert np.all(cut.eval["precision"][:, :, 0, 0] == 0)
    kept = run(gts, dts, [image(1)], max_dets=301)
    assert np.all(kept.eval["recall"][:, 0, 0] == 1)
    assert np.all(kept.eval["precision"][:, :, 0, 0] == ONE)


def test_an_unlisted_category_changes_no_number_but_takes_a_slot_of_the_cut():
    gts = [gt(1, 1, BOX)]
    base = [dt(1, 1, BOX, 0.5)]
    extra = [dt(1, 3, FAR, 0.9)]        # category 3: neither positive nor negative for image 1
    a = run(gts, base, [image(1)], max_dets=2)
    b = run(gts, extra + base, [image(1)], max_dets=2)
    for name in ("precision", "recall"):
        assert np.array_equal(a.eval[name], b.eval[name])
    assert a.results == b.results and a.results["AP"] == ONE
    c = run(gts, extra + base, [image(1)], max_dets=1)
    assert np.all(c.eval["recall"][:, 0, 0] == 0)
    assert c.results["AP"] == 0


def test_a_negative_category_detection_is_a_false_positive():
    gts = [gt(1, 1, BOX), gt(2, 2, BOX)]
    dts = [dt(1, 1, BOX, 0.9), dt(1, 2, FAR, 0.8), dt(2, 2, BOX, 0.5)]
    neg = run(gts, dts, [image(1, neg=[2]), image(2)])
    assert np.all(neg.eval["precision"][:, :, 1, 0] == 0.5)
    dropped = run(gts, dts, [image(1), image(2)])
    assert np.all(dropped.eval["precision"][:, :, 1, 0] == ONE)


def test_not_exhaustive_ignores_unmatched_detections_only():
    gts = [gt(1, 1, BOX)]
    dts = [dt(1, 1, FAR, 0.95), dt(1, 1, BOX, 0.9)]
    nel = run(gts, dts, [image(1, nel=[1])])
    assert np.all(nel.eval["precision"][:, :, 0, 0] == ONE)
    assert np.all(nel.eval["recall"][:, 0, 0] == 1)      # the matched one is still a TP
    e = nel.eval_imgs[0]
    assert e["dt_ignore"][:, 0].all() and not e["dt_ignore"][:, 1].any()
    exhaustive = run(gts, dts, [image(1)])
    assert np.all(exhaustive.eval["precision"][:, :, 0, 0] == 0.5)


def test_a_crowd_annotation_is_an_ordinary_instance():
    m = np.zeros((20, 20), bool)
    m[2:12, 2:12] = True
    half = m.copy()
    half[2:12, 7:12] = False
    g = [{"image_id": 1, "category_id": 1, "mask": m, "iscrowd": 1, "area": 100.0}]
    d = [{"image_id": 1, "category_id": 1, "mask": half, "score": 0.9}]
    p = lo.Params("segm")
    ev = lo.LVISEvalOracle(g, d, [image(1)], CATS, "segm", p)
    ev.run()
    # a crowd's IoU would be 50 / 50 = 1; an ordinary instance's is 50 / 100
    assert ev.ious[1, 1][0, 0] == 0.5
    assert np.all(ev.eval["recall"][:1, 0, 0] == 1) and np.all(ev.eval["recall"][1:, 0, 0] == 0)
    coco = co.COCOevalOracle(g, d)
    coco.evaluate()
    coco.accumulate()
    assert coco.ious[1, 1][0, 0] == 1.0
    assert np.all(coco.eval["recall"] == -1)      # COCO: the only instance is a crowd, ignored


def test_frequency_groups_and_an_empty_group():
    cats = [{"id": 1, "frequency": "r"}, {"id": 2, "frequency": "f"}]
    gts = [gt(1, 1, BOX), gt(2, 2, BOX)]
    dts = [dt(1, 1, BOX, 0.9), dt(1, 2, FAR, 0.8), dt(2, 2, BOX, 0.5)]
    ev = run(gts, dts, [image(1, neg=[2]), image(2)], cats=cats)
    assert ev.freq_groups == [[0], [], [1]]
    assert ev.results["APr"] == ONE and ev.results["APf"] == 0.5 and ev.results["APc"] == -1
    assert ev.results["AP"] == pytest.approx(0.75)
    assert list(ev.results) == ["AP", "AP50", "AP75", "APs", "APm", "APl", "APr", "APc", "APf",
                                "AR@300", "ARs@300", "ARm@300", "ARl@300"]
    with redirect_stdout(io.StringIO()) as out:
        ev.print_results()
    lines = out.getvalue().splitlines()
    assert lines[0] == (" Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=300 "
                        "catIds=all] = 0.750")
    assert lines[7] == (" Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=300 "
                        "catIds=  c] = -1.000")
    assert lines[10] == (" Average Recall     (AR) @[ IoU=0.50:0.95 | area=     s | maxDets=300 "
                         "catIds=all] = 1.000")


def test_nan_scores_sort_last_in_the_cut():
    kept = lo.limit_dets_per_image([dt(1, 1, BOX, s) for s in (np.nan, 0.2, 0.7, 0.2)], 3)
    assert [d["id"] for d in kept] == [2, 1, 3]


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_cross_check_with_cocoeval(seed):
    """No crowds, every category without ground truth in an image listed as negative, nothing
    not exhaustive, at most 100 detections per image, the same category ids: LVISEval's
    precision and recall are COCOeval's at maxDets 100, bit for bit."""
    from test_host_cocoeval import _random_dataset

    gts, dts = _random_dataset(seed)
    for g in gts:
        g["iscrowd"] = 0
    cat_ids = sorted({g["category_id"] for g in gts})
    img_ids = sorted({g["image_id"] for g in gts} | {d["image_id"] for d in dts})
    cats = [{"id": c, "frequency": "rcf"[c % 3]} for c in cat_ids]
    images = [image(i, neg=[c for c in cat_ids
                            if not any(g["image_id"] == i and g["category_id"] == c for g in gts)])
              for i in img_ids]
    assert max(sum(d["image_id"] == i for d in dts) for i in img_ids) <= 100
    ev = lo.LVISEvalOracle(gts, dts, images, cats, "segm")
    ev.run()
    p = co.Params()
    p.catIds = list(cat_ids)
    coco = co.COCOevalOracle(gts, dts, p)
    coco.evaluate()
    coco.accumulate()
    for name, sl in (("precision", np.s_[..., -1]), ("recall", np.s_[..., -1])):
        want = coco.eval[name][sl]
        assert ev.eval[name].shape == want.shape
        assert np.array_equal(ev.eval[name].view(np.uint64), np.ascontiguousarray(want).view(np.uint64))
    assert (ev.eval["precision"] > 0).any() and (ev.eval["precision"] < 1).any()
