"""CPU tests of the host half of evaluate.LVISEvalSegm / LVISEvalBbox: the vectorised accumulate,
summarize and print_results against the restated LVISEval loop (tests/lvis_oracle.py) on records
built from its per-image results, the status table of the federated filter, the not-exhaustive
rule on downloaded flags, and the ValueError cases."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest

import lvis_oracle as lo
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import evaluate


def random_lvis(seed, n_img=16, n_cat=7, max_dt=14, max_gt=6, freqs="rcf"):
    """Random LVIS-like boxes: neg and not-exhaustive lists, detections of unlisted categories,
    score ties and NaN scores, images without detections or lists."""
    rng = np.random.default_rng(seed)
    cats = [{"id": 10 + c, "frequency": freqs[c % len(freqs)]} for c in range(n_cat)]
    cat_ids = [c["id"] for c in cats]
    gts, dts, images = [], [], []
    for img in rng.permutation(np.arange(1, n_img + 1) * 5):
        img = int(img)
        mine = []
        for _ in range(rng.integers(0, max_gt + 1)):
            x, y = rng.integers(0, 40, size=2)
            bb = [float(x), float(y), float(rng.integers(1, 20)), float(rng.integers(1, 20))]
            g = {"image_id": img, "category_id": int(rng.choice(cat_ids)), "bbox": bb,
                 "iscrowd": int(rng.random() < 0.2),
                 "area": float(rng.choice([bb[2] * bb[3], 30.0, 150.0]))}
            gts.append(g)
            mine.append(g)
        pos = {g["category_id"] for g in mine}
        rest = [c for c in cat_ids if c not in pos]
        neg = [c for c in rest if rng.random() < 0.5] if rng.random() < 0.8 else []
        nel = [c for c in pos if rng.random() < 0.3]
        images.append({"id": img, "height": 64, "width": 64, "neg_category_ids": neg,
                       "not_exhaustive_category_ids": nel})
        for _ in range(rng.integers(0, max_dt + 1)):
            s = float(rng.choice([0.1, 0.5, 0.5, 0.9, np.nan, rng.random()]))
            if mine and rng.random() < 0.6:
                g = mine[rng.integers(len(mine))]
                bb = [v + float(rng.integers(-2, 3)) for v in g["bbox"][:2]] + g["bbox"][2:]
                dts.append({"image_id": img, "category_id": g["category_id"], "bbox": bb,
                            "score": s})
                continue
            x, y = rng.integers(0, 40, size=2)
            bb = [float(x), float(y), float(rng.integers(1, 20)), float(rng.integers(1, 20))]
            dts.append({"image_id": img, "category_id": int(rng.choice(cat_ids + [99])),
                        "bbox": bb, "score": s})
    return gts, dts, images, cats


def run_oracle(gts, dts, images, cats, max_dets=300, **params):
    p = lo.Params("bbox")
    p.max_dets = max_dets
    for k, v in params.items():
        setattr(p, k, v)
    ev = lo.LVISEvalOracle(gts, dts, images, cats, "bbox", p)
    ev.run()
    with redirect_stdout(io.StringIO()) as out:
        ev.print_results()
    ev.printed = out.getvalue()
    return ev


def product_from_oracle(ev, images, cats):
    """An LVISEvalBbox holding the records the device would have produced for ev's images (its
    eval_imgs' matches and ignore flags), in an image order other than the id order."""
    p = ev.params
    out = evaluate.LVISEvalBbox(cats, images, iou_thrs=p.iou_thrs, max_dets=p.max_dets,
                                area_rng=p.area_rng, area_rng_lbl=p.area_rng_lbl)
    I0, A0, T = len(p.img_ids), len(p.area_rng), len(p.iou_thrs)
    for pos, img in enumerate(reversed(p.img_ids)):
        out._img_index[img] = pos
    img, cat, rank, score, tp, ig = [], [], [], [], [], []
    for k, c in enumerate(p.cat_ids):
        for i, im in enumerate(p.img_ids):
            es = [ev.eval_imgs[k * A0 * I0 + a * I0 + i] for a in range(A0)]
            if es[0] is None:
                continue
            D = len(es[0]["dt_scores"])
            img += [out._img_index[im]] * D
            cat += [out._cat_index[c]] * D
            rank += list(range(D))
            score += es[0]["dt_scores"]
            tp.append(np.stack([e["dt_matches"].T > -1 for e in es], axis=1))
            ig.append(np.stack([e["dt_ignore"].T.astype(bool) for e in es], axis=1))
    out._dets.append((np.array(img, np.int64), np.array(cat, np.int32), np.array(rank, np.int32),
                      np.array(score, np.float64), np.concatenate(tp + [np.zeros((0, A0, T), bool)]),
                      np.concatenate(ig + [np.zeros((0, A0, T), bool)])))
    g = [x for x in ev.gts_in if x["category_id"] in p.cat_ids]
    nonig = np.array([[lo_ <= x["area"] <= hi for lo_, hi in p.area_rng] for x in g],
                     bool).reshape(-1, A0)
    out._gts.append((np.array([out._img_index[x["image_id"]] for x in g], np.int64),
                     np.array([out._cat_index[x["category_id"]] for x in g], np.int32), nonig))
    out._sync_params()
    out.params.rec_thrs = p.rec_thrs
    return out


def same(got, ev):
    for name in ("precision", "recall"):
        a, b = got.eval[name], ev.eval[name]
        assert a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64)), name
    assert got.eval["counts"] == ev.eval["counts"]
    assert list(got.results) == list(ev.results)
    for k in ev.results:
        assert np.float64(got.results[k]).view(np.uint64) == \
            np.float64(ev.results[k]).view(np.uint64), k
    with redirect_stdout(io.StringIO()) as out:
        got.print_results()
    assert out.getvalue() == ev.printed


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("max_dets,freqs", [(300, "rcf"), (6, "rcf"), (3, "rf")])
def test_accumulate_summarize_equal_the_loop(seed, max_dets, freqs):
    gts, dts, images, cats = random_lvis(seed, freqs=freqs)
    ev = run_oracle(gts, dts, images, cats, max_dets)
    got = product_from_oracle(ev, images, cats)
    got.run()
    same(got, ev)
    assert (ev.eval["precision"] > 0).any()
    if freqs == "rf":
        assert ev.results["APc"] == -1


def test_image_and_category_subsets():
    gts, dts, images, cats = random_lvis(7)
    ev = run_oracle(gts, dts, images, cats, 8)
    got = product_from_oracle(ev, images, cats)
    keep_imgs, keep_cats = ev.params.img_ids[::2], ev.params.cat_ids[1:]
    sub = run_oracle(gts, dts, images, cats, 8, img_ids=list(keep_imgs), cat_ids=list(keep_cats))
    got.params.img_ids, got.params.cat_ids = list(keep_imgs), list(keep_cats)
    got.accumulate()
    got.summarize()
    same(got, sub)


def test_default_params_are_lvis_apis():
    p, q = evaluate.LVISEvalSegm([{"id": 3, "frequency": "f"}, {"id": 1, "frequency": "r"}],
                                 []).params, lo.Params()
    for name in ("iou_thrs", "rec_thrs", "max_dets", "area_rng", "area_rng_lbl", "use_cats",
                 "img_count_lbl"):
        assert np.array_equal(getattr(p, name), getattr(q, name)), name
    assert p.cat_ids == [1, 3] and p.img_ids == [] and p.iou_type == "segm"


CATS = [{"id": 1, "frequency": "r"}, {"id": 5, "frequency": "c"}, {"id": 9, "frequency": "f"}]
IMAGES = [{"id": 7, "height": 4, "width": 6, "neg_category_ids": [5, 42],
           "not_exhaustive_category_ids": [1]},
          {"id": 8, "height": 4, "width": 6, "neg_category_ids": [],
           "not_exhaustive_category_ids": []}]


def test_status_table():
    ev = evaluate.LVISEvalBbox(CATS, IMAGES)
    st = ev.status_table([7, 8], [np.array([0, 2, 0, -1], np.int32), np.array([1], np.int32)])
    P, Ng, X = N.MRX_LVIS_POSITIVE, N.MRX_LVIS_NEGATIVE, N.MRX_LVIS_NOT_EXHAUSTIVE
    assert st.dtype == np.uint8
    assert st.tolist() == [[P | X, Ng, P], [0, P, 0]]
    assert N.MRX_LVIS_EVALUATED == P | Ng


def test_not_exhaustive_rule_on_downloaded_flags():
    status = np.array([[N.MRX_LVIS_POSITIVE | N.MRX_LVIS_NOT_EXHAUSTIVE, N.MRX_LVIS_NEGATIVE]],
                      np.uint8)
    cat = np.array([[0, 0, 1, -1]], np.int32)
    match = np.array([[[[-1, 3, -1, -1]], [[-1, -1, -1, -1]]]], np.int32)     # [A=1, T=2, 1, 4]
    cat[0, 3] = 1 << 30                    # not kept: a value the device never wrote
    res = {"cat": cat, "match": match, "ignore": np.zeros(match.shape, bool),
           "keep": np.array([[True, True, True, False]])}
    evaluate.LVISEvalBbox.not_exhaustive(res, status)
    assert res["ignore"][0, :, 0].tolist() == [[True, False, False, False],
                                                [True, True, False, False]]


def test_record_applies_the_not_exhaustive_rule():
    """_record on a downloaded batch: image 7 lists category 1 (dense 0) as not exhaustive."""
    ev = evaluate.LVISEvalBbox(CATS, IMAGES, area_rng=[[0, 1e10]], area_rng_lbl=["all"],
                               iou_thrs=[0.5])
    res = {"cat": np.array([[0, 0, 1], [0, 2, -1]], np.int32),
           "rank": np.array([[0, 1, 0], [0, 0, 0]], np.int32),
           "keep": np.array([[True, True, True], [True, True, False]]),
           "score": np.array([[0.9, 0.8, 0.7], [0.6, 0.5, 0.0]]),
           "match": np.array([[[[2, -1, -1], [-1, -1, -1]]]], np.int32),
           "ignore": np.zeros((1, 1, 2, 3), bool)}
    cats = [np.array([0, 2, 0], np.int32), np.array([1], np.int32)]
    ev._record([7, 8], res, cats, [np.zeros(3, np.uint8), np.zeros(1, np.uint8)],
               [np.array([5.0, 50.0, 500.0]), np.array([1.0])])
    img, cat, rank, score, tp, ig = ev._dets[0]
    assert img.tolist() == [0, 0, 0, 1, 1] and cat.tolist() == [0, 0, 1, 0, 2]
    assert tp[:, 0, 0].tolist() == [True, False, False, False, False]
    # image 7, category 1: the matched one counts, the unmatched one is ignored; image 8 lists none
    assert ig[:, 0, 0].tolist() == [False, True, False, False, False]
    assert ev._gts[0][2].ravel().tolist() == [True] * 4
    assert ev.params.img_ids == [7, 8]


RLE = {"size": [4, 6], "counts": b"0j0"}


@pytest.mark.parametrize("call,msg", [
    (lambda: evaluate.LVISEvalSegm(CATS, IMAGES).add_results([], [[]], [3]),
     "image 3 is not one of the dataset's images"),
    (lambda: evaluate.LVISEvalBbox(CATS, IMAGES).add_results([], [[]], [3]),
     "image 3 is not one of the dataset's images"),
    (lambda: evaluate.LVISEvalSegm(CATS, [{"id": 4, "height": 1, "width": 1,
                                           "neg_category_ids": []}]),
     r"image 4: no \['not_exhaustive_category_ids'\]"),
    (lambda: evaluate.LVISEvalSegm(CATS + [{"id": 2, "frequency": "x"}], IMAGES),
     "category 2: frequency 'x' is not one of"),
    (lambda: evaluate.LVISEvalBbox(CATS, IMAGES, max_dets=0), r"max_dets = 0 \(need >= 1\)"),
    (lambda: evaluate.LVISEvalSegm(CATS, IMAGES).add_results(
        [], [[{"category_id": 1, "segmentation": RLE, "area": 3.0, "ignore": 1, "id": 4}]], [7]),
     r"image 7, annotation 0 \(id 4\): 'ignore' annotations are not supported"),
    (lambda: evaluate.LVISEvalBbox(CATS, IMAGES).add_results(
        [], [[{"category_id": 1, "bbox": [0, 0, 1, 1], "area": 1.0, "ignore": True}]], [8]),
     r"image 8, annotation 0: 'ignore' annotations are not supported"),
    (lambda: evaluate.LVISEvalSegm(CATS, IMAGES).add_results(
        [{"image_id": 7, "category_id": 1, "score": 1.0,
          "segmentation": {"size": [5, 6], "counts": b"0m0"}}], [[]], [7]),
     r"image 7: RLE sizes .* differ"),
    (lambda: evaluate.LVISEvalSegm(CATS, IMAGES, cat_ids=[1, 2]), r"cat_ids \[2\] are not"),
])
def test_value_errors(call, msg):
    with pytest.raises(ValueError, match=msg):
        call()


@pytest.mark.parametrize("name,value", [("iou_thrs", np.array([0.5])),
                                        ("area_rng", [[0, 1e10]]), ("max_dets", 100)])
def test_params_frozen_after_the_first_batch(name, value):
    ev = evaluate.LVISEvalSegm(CATS, IMAGES)
    ev._freeze()
    setattr(ev.params, name, value)
    with pytest.raises(ValueError, match="changed after the first batch"):
        ev.accumulate()


def test_summarize_before_accumulate():
    with pytest.raises(RuntimeError, match="accumulate"):
        evaluate.LVISEvalBbox(CATS, IMAGES).summarize()
