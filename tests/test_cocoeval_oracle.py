"""The COCOeval "segm" restatement (tests/cocoeval_oracle.py) on answers worked by hand."""
import io
from contextlib import redirect_stdout

import numpy as np

import cocoeval_oracle as co

EPS = np.spacing(1)
# pycocotools' precision of a true positive with no false positive before it: tp / (tp + eps)
P1 = 1 / (1 + EPS)


def sq(y1, x1, y2, x2, hw=(40, 40)):
    m = np.zeros(hw, bool)
    m[y1:y2, x1:x2] = True
    return m


def gt(img, cat, mask, crowd=0, area=None):
    return {"image_id": img, "category_id": cat, "mask": mask, "iscrowd": crowd,
            "area": float(mask.sum()) if area is None else area}


def dt(img, cat, mask, score):
    return {"image_id": img, "category_id": cat, "mask": mask, "score": score}


def run(gts, dts, **params):
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


def test_one_perfect_detection():
    m = sq(5, 5, 15, 15)
    ev = run([gt(1, 1, m)], [dt(1, 1, m, 0.9)])
    pr = ev.eval["precision"]
    assert (pr[:, :, 0, 0, :] == P1).all() and (pr[:, :, 0, 1, :] == P1).all()
    assert (pr[:, :, 0, 2:, :] == -1).all()             # no medium or large ground truth
    assert (ev.eval["recall"][:, 0, :2, :] == 1).all()
    assert (ev.eval["scores"][:, :, 0, 0, :] == 0.9).all()
    want = [P1, P1, P1, P1, -1, -1, 1, 1, 1, 1, -1, -1]
    assert np.allclose(ev.stats, want, rtol=0, atol=1e-15)    # the means round to 1 here
    assert ev.printed.splitlines()[0] == \
        " Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = 1.000"


def test_detections_on_a_crowd_region_are_ignored():
    crowd = sq(0, 0, 20, 20)
    ev = run([gt(1, 1, crowd, crowd=1)], [dt(1, 1, sq(0, 0, 10, 10), 0.9),
                                          dt(1, 1, sq(10, 10, 20, 20), 0.8)])
    e = ev.evalImgs[0]
    assert (e["dtMatches"] == 0).all() and e["dtIgnore"].all()    # both on the one crowd region
    assert (ev.eval["precision"] == -1).all() and (ev.eval["recall"] == -1).all()   # npig = 0
    assert (ev.stats == -1).all()


def test_crowd_iou_is_intersection_over_detection_area():
    crowd, d = sq(0, 0, 10, 10), sq(5, 0, 15, 5)          # 25 of the detection's 50 inside
    ev = run([gt(1, 1, crowd, crowd=1), gt(1, 1, crowd)], [dt(1, 1, d, 0.9)])
    assert ev.ious[1, 1][0, 0] == 25 / 50
    assert ev.ious[1, 1][0, 1] == 25 / (50 + 100 - 25)
    assert co.rle_iou(d, sq(20, 20, 30, 30), 1) == 0.0     # i = 0: 0, not NaN
    assert co.rle_iou(np.zeros((4, 4), bool), np.zeros((4, 4), bool), 0) == 0.0


def test_area_1024_is_small_and_medium():
    m = sq(0, 0, 32, 32)
    ev = run([gt(1, 1, m, area=1024.0)], [dt(1, 1, m, 0.9)])
    r = ev.eval["recall"][:, 0, :, 2]
    assert (r[:, :3] == 1).all() and (r[:, 3] == -1).all()
    ev = run([gt(1, 1, m, area=1024.5)], [dt(1, 1, m, 0.9)])
    assert (ev.eval["recall"][:, 0, 1, 2] == -1).all()     # above small; the detection ignored too


def test_cross_image_ties_go_in_image_id_order():
    a, b = sq(0, 0, 10, 10), sq(20, 20, 30, 30)
    # image 2 is listed first; its detection misses, image 1's hits, both score 0.5
    gts = [gt(2, 1, a), gt(1, 1, a)]
    dts = [dt(2, 1, b, 0.5), dt(1, 1, a, 0.5)]
    ev = run(gts, dts)
    pr = ev.eval["precision"][0, :, 0, 0, 2]
    # sorted by image id: tp = [1, 1], fp = [0, 1]: rc = [.5, .5], pr = [P1, .5]
    assert np.array_equal(pr, [P1] * 51 + [0] * 50)
    assert ev.eval["recall"][0, 0, 0, 2] == 0.5


def test_max_dets_cuts_per_image_and_category():
    a, b = sq(0, 0, 10, 10), sq(20, 20, 30, 30)
    gts = [gt(1, 1, a), gt(1, 2, b)]
    dts = [dt(1, 1, b, 0.9), dt(1, 1, a, 0.8), dt(1, 2, b, 0.95)]
    ev = run(gts, dts, maxDets=[1, 2, 100])
    rec = ev.eval["recall"][0, :, 0, :]
    assert np.array_equal(rec[0], [0, 1, 1])      # category 1: its best detection misses
    assert np.array_equal(rec[1], [1, 1, 1])      # category 2's own cut is not shared


def test_iou_threshold_one_still_matches_a_perfect_mask():
    m = sq(3, 3, 9, 13)
    ev = run([gt(1, 1, m)], [dt(1, 1, m, 0.9)], iouThrs=np.array([0.5, 1.0]))
    assert (ev.eval["recall"][:, 0, 0, 2] == 1).all()


def test_three_detection_curve():
    a, b, c = sq(0, 0, 10, 10), sq(20, 20, 30, 30), sq(0, 20, 10, 30)
    gts = [gt(1, 1, a), gt(1, 1, b)]
    dts = [dt(1, 1, a, 0.9), dt(1, 1, c, 0.8), dt(1, 1, b, 0.7)]
    ev = run(gts, dts)
    # tp = [1, 1, 2], fp = [0, 1, 1], npig = 2: rc = [.5, .5, 1], pr = [P1, 1/2, 2/3] with
    # 2 + eps == 2 and 3 + eps == 3; envelope [P1, 2/3, 2/3]; recall .00-.50 -> index 0,
    # .51-1.00 -> index 2
    want = np.array([P1] * 51 + [2 / 3] * 50)
    for t in range(10):
        assert np.array_equal(ev.eval["precision"][t, :, 0, 0, 2], want)
        assert np.array_equal(ev.eval["scores"][t, :, 0, 0, 2], [0.9] * 51 + [0.7] * 50)
        assert ev.eval["recall"][t, 0, 0, 2] == 1.0
    assert abs(ev.stats[0] - np.mean(want)) < 1e-15


def test_category_without_ground_truth_is_excluded():
    m = sq(5, 5, 15, 15)
    ev = run([gt(1, 1, m)], [dt(1, 1, m, 0.9), dt(1, 2, m, 0.8)], catIds=[1, 2])
    assert (ev.eval["precision"][:, :, 1] == -1).all() and (ev.eval["recall"][:, 1] == -1).all()
    one = run([gt(1, 1, m)], [dt(1, 1, m, 0.9)])
    assert np.array_equal(ev.stats, one.stats)
