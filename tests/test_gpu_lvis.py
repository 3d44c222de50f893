"""LVIS evaluation on the device (mrx_lvis_ranks and evaluate.LVISEvalSegm / LVISEvalBbox): the
per-image cut and federated filter exactly as the restated LVISResults / LVISEval
(tests/lvis_oracle.py) apply them, and everything after them -- IoUs bit for bit, match and ignore
flags, the accumulated arrays and results -- equal to the oracle run on what
unmold_detections_batch returns."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

import lvis_oracle as lo
import polygon_oracle as po
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate, synth

from helpers import item_of

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------------------- ranks
def expected_ranks(cls, scores, n, class_map, status, max_det):
    """cat, rank, walk and keep of one image from the oracle's cut (limit_dets_per_image) and
    _prepare's filter."""
    C, K = class_map.size, status.size
    s = scores[:n].astype(np.float64)
    cat = np.array([class_map[c] if 0 <= c < C else -1 for c in cls[:n]], np.int64)
    walk = np.argsort(np.where(np.isnan(s), np.inf, -s), kind="mergesort")   # NaN last, stable
    pos = np.empty(n, np.int64)
    pos[walk] = np.arange(n)
    rank = np.array([int(np.sum((cat[walk[:pos[i]]] == cat[i]))) for i in range(n)], np.int64)
    cut = {d["id"] for d in lo.limit_dets_per_image(
        [{"image_id": 0, "score": float(v)} for v in s], max_det)}
    keep = np.array([i in cut and 0 <= cat[i] < K and bool(status[cat[i]] & N.MRX_LVIS_EVALUATED)
                     for i in range(n)], bool)
    return cat, rank, walk, keep


RANK_CASES = [  # (seed, B, R, K, C, max_det, score dtype)
    (1, 4, 300, 1203, 1300, 300, np.float32),
    (2, 4, 300, 1203, 1300, 1, np.float32),
    (3, 5, 300, 1203, 1300, 57, np.float64),
    (4, 3, 64, 2000, 2100, 64, np.float64),
    (5, 3, 64, 2000, 2100, 500, np.float32),
    (6, 2, 700, 1203, 1210, 300, np.float32),
]


@pytest.mark.parametrize("case", RANK_CASES, ids=lambda c: f"seed{c[0]}-R{c[2]}-K{c[3]}-m{c[5]}")
def test_lvis_ranks_equal_the_cut_and_filter(cuda_device, case):
    seed, B, R, K, C, max_det, sdt = case
    rng = np.random.default_rng(seed)
    counts = rng.integers(R // 2, R + 1, size=B).astype(np.int32)
    counts[0] = R
    counts[-1] = 0                                     # an image without predictions
    cls = rng.integers(-2, C + 3, size=(B, R)).astype(np.int32)
    scores = np.round(rng.random((B, R)), 2).astype(sdt)    # ties across categories
    scores[rng.random((B, R)) < 0.03] = np.nan
    class_map = rng.integers(0, K + 5, size=C).astype(np.int32)     # some at or above K
    class_map[rng.random(C) < 0.1] = -1
    status = rng.integers(0, 8, size=(B, K)).astype(np.uint8)
    status[1 % B] = 0                                  # an image without lists or ground truth
    dev = torch.device("cuda")
    d = {k: torch.from_numpy(v).to(dev) for k, v in
         dict(cls=cls, scores=scores, counts=counts, map=class_map, status=status).items()}
    out = {k: torch.full((B, R), -7, dtype=torch.int32, device=dev) for k in ("cat", "rank", "walk")}
    keep = torch.full((B, R), 9, dtype=torch.uint8, device=dev)
    lib = N.load()
    N.check(lib.mrx_lvis_ranks(
        d["cls"], d["scores"], N.MRX_F64 if sdt == np.float64 else N.MRX_F32, d["counts"],
        d["map"], C, d["status"], K, max_det, out["cat"], out["rank"], keep, out["walk"], B, R,
        N.stream_ptr(None)), "mrx_lvis_ranks")
    got = {k: v.cpu().numpy() for k, v in out.items()}
    got_keep = keep.cpu().numpy()
    kept_at_cut = 0
    for b in range(B):
        n = int(counts[b])
        cat, rank, walk, want_keep = expected_ranks(cls[b], scores[b], n, class_map, status[b],
                                                    max_det)
        cat = np.where(cat < 0, -1, cat)
        assert np.array_equal(got["cat"][b, :n], cat), b
        assert np.array_equal(got["rank"][b, :n], rank), b
        assert np.array_equal(got["walk"][b, :n], walk), b
        assert np.array_equal(got_keep[b, :n] != 0, want_keep), b
        assert (got_keep[b, n:] == 9).all() and (got["cat"][b, n:] == -7).all()
        kept_at_cut += int(want_keep.sum())
    assert kept_at_cut > 0


def test_lvis_ranks_argument_checks(cuda_device):
    lib = N.load()
    t = torch.zeros(16, dtype=torch.int32, device="cuda")
    p = t.data_ptr()
    base = [p, p, N.MRX_F32, p, p, 4, p, 3, 10, p, p, p, p, 1, 4, N.stream_ptr(None)]
    assert lib.mrx_lvis_ranks(*base) == N.MRX_OK
    for k, bad in ((6, None), (7, 0), (8, 0), (13, -1), (14, 0), (2, 5)):
        args = list(base)
        args[k] = bad
        assert lib.mrx_lvis_ranks(*args) < 0, k
    args = list(base)
    args[13] = 0
    assert lib.mrx_lvis_ranks(*args) == N.MRX_OK


# ----------------------------------------------------------------------------- evaluators
class CaptureSegm(evaluate.LVISEvalSegm):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.batches = []

    def _record(self, image_ids, res, *rest):
        self.batches.append((list(image_ids), res))
        super()._record(image_ids, res, *rest)


class CaptureBbox(evaluate.LVISEvalBbox):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.batches = []

    def _record(self, image_ids, res, *rest):
        self.batches.append((list(image_ids), res))
        super()._record(image_ids, res, *rest)


CLASSES = 6
CMAP = [0, 11, 12, 13, 14, 999]            # class 5 is not a category of the dataset
CATS = [{"id": 11, "frequency": "r"}, {"id": 12, "frequency": "c"}, {"id": 13, "frequency": "f"},
        {"id": 14, "frequency": "f"}, {"id": 15, "frequency": "c"}]
STREAM = [  # (image ids, shapes, n, R)
    ([30, 10], [(160, 200), (120, 96)], 300, 300),
    ([20, 5], [(97, 203), (64, 64)], 150, 300),
]


def make_batch(seed, shapes, n, R, cross_check=False):
    """items, annotation lists (polygon ground truth from jittered predicted boxes, a box-list
    one, crowds that LVIS ignores), the ground-truth masks and the LVIS image dicts."""
    rng = np.random.default_rng(seed)
    ims = [synth.make_image(rng, hw, n, num_classes=CLASSES, max_instances=R,
                            **({} if min(hw) > 64 else dict(min_box=1, max_box_frac=1.0)))
           for hw in shapes]
    for im in ims:
        im.detections[:im.n_valid, 5] = np.round(im.detections[:im.n_valid, 5], 1)
    items = [item_of(im, np.float32) for im in ims]
    preds = api_utils.unmold_detections_batch(items)
    anns, masks = [], []
    for (boxes, cls, _, _), im in zip(preds, ims):
        H, W = im.original_image_shape[:2]
        a, ms = [], []
        for k in range(0, cls.shape[0], 3):
            y1, x1, y2, x2 = (int(v) + int(s) for v, s in zip(boxes[k], rng.integers(-3, 4, 4)))
            y1, y2 = min(y1, y2), max(y1, y2) + 1
            x1, x2 = min(x1, x2), max(x1, x2) + 1
            poly = [float(x1), float(y1), float(x2), float(y1 + 2), float(x2 - 3), float(y2),
                    float(x1 + 1), float(y2 - 1)]
            c = int(cls[k]) if rng.random() > 0.15 else int(rng.integers(1, CLASSES))
            seg = [poly] if k % 7 else [[float(x1), float(y1), float(x2 - x1), float(y2 - y1)]]
            m = po.ann_to_mask(seg, H, W).astype(bool)
            a.append({"category_id": CMAP[c], "segmentation": seg,
                      "iscrowd": 0 if cross_check else int(rng.random() < 0.1),
                      "area": float(rng.choice([m.sum(), 500.0, 5000.0])), "id": len(a) + 1,
                      "bbox": [float(x1), float(y1), float(x2 - x1), float(y2 - y1)]})
            ms.append(m)
        anns.append(a)
        masks.append(ms)
    return items, anns, masks, preds


def lvis_images(rng, ids, anns, cross_check=False):
    out = []
    cat_ids = [c["id"] for c in CATS]
    for i, a in zip(ids, anns):
        pos = sorted({x["category_id"] for x in a if x["category_id"] in cat_ids})
        rest = [c for c in cat_ids if c not in pos]
        neg = rest if cross_check else [c for c in rest if rng.random() < 0.5]
        nel = [] if cross_check else [c for c in pos if rng.random() < 0.4]
        out.append({"id": i, "height": 0, "width": 0, "neg_category_ids": neg,
                    "not_exhaustive_category_ids": nel})
    return out


def stream(seed, stream_def=STREAM, cross_check=False):
    rng = np.random.default_rng(seed + 1000)
    batches, images = [], []
    for s, (ids, shapes, n, R) in enumerate(stream_def):
        items, anns, masks, preds = make_batch(seed + s, shapes, n, R, cross_check)
        ims = lvis_images(rng, ids, anns, cross_check)
        for im, (H, W) in zip(ims, shapes):
            im["height"], im["width"] = H, W
        images += ims
        batches.append((ids, items, anns, masks, preds))
    return batches, images


def oracle_inputs(batches, iou_type):
    gts, dts, gmap, dmap = [], [], {}, {}
    for ids, items, anns, masks, preds in batches:
        for img, a, ms, (boxes, cls, scores, pm) in zip(ids, anns, masks, preds):
            for j, (ann, m) in enumerate(zip(a, ms)):
                gmap[len(gts)] = (img, j)
                g = {"image_id": img, "category_id": ann["category_id"], "area": ann["area"],
                     "iscrowd": ann["iscrowd"]}
                g.update(mask=m) if iou_type == "segm" else g.update(bbox=ann["bbox"])
                gts.append(g)
            for i in range(cls.shape[0]):
                dmap[len(dts)] = (img, i)
                d = {"image_id": img, "category_id": CMAP[int(cls[i])], "score": float(scores[i])}
                if iou_type == "segm":
                    d["mask"] = pm[:, :, i]
                else:
                    y1, x1, y2, x2 = (int(v) for v in boxes[i])
                    d["bbox"] = [x1, y1, x2 - x1, y2 - y1]
                dts.append(d)
    return gts, dts, gmap, dmap


def run_oracle(gts, dts, images, iou_type, max_dets):
    p = lo.Params(iou_type)
    p.max_dets = max_dets
    ev = lo.LVISEvalOracle(gts, dts, images, CATS, iou_type, p)
    ev.run()
    with redirect_stdout(io.StringIO()) as out:
        ev.print_results()
    ev.printed = out.getvalue()
    return ev


def check_pairs(ev, got, gmap, dmap):
    where = {}
    for ids, res in got.batches:
        for b, img in enumerate(ids):
            where[img] = (b, res)
    inv_cat = {d: c for c, d in got._cat_index.items()}
    n_iou = n_flags = n_kept = 0
    for (img, cat), dts in ev._dts.items():
        b, res = where[img]
        order = np.argsort([-d["score"] for d in dts], kind="mergesort")
        ious = ev.ious[img, cat]
        d_iou = res["d_iou"][b].cpu().numpy()
        for di, o in enumerate(order):
            i = dmap[dts[o]["id"]][1]
            assert res["keep"][b, i] and res["rank"][b, i] == di, (img, cat, i)
            assert inv_cat[res["cat"][b, i]] == cat
            n_kept += 1
            for gi, g in enumerate(ev._gts[img, cat]):
                j = gmap[g["id"]][1]
                assert d_iou[i, j].view(np.uint64) == np.float64(ious[di, gi]).view(np.uint64), \
                    (img, cat, i, j, d_iou[i, j], ious[di, gi])
                n_iou += 1
    assert n_kept == sum(int(res["keep"].sum()) for _, res in got.batches)
    p = ev.params
    nI, nA = len(p.img_ids), len(p.area_rng)
    for k, cat in enumerate(p.cat_ids):
        for a in range(nA):
            for ii, img in enumerate(p.img_ids):
                e = ev.eval_imgs[k * nA * nI + a * nI + ii]
                if e is None:
                    continue
                b, res = where[img]
                for di, did in enumerate(e["dt_ids"]):
                    i = dmap[did][1]
                    want = [gmap[g][1] if g > -1 else -1 for g in e["dt_match_ids"][:, di]]
                    assert np.array_equal(res["match"][a, :, b, i], want), (img, cat, a, i)
                    assert np.array_equal(res["ignore"][a, :, b, i], e["dt_ignore"][:, di] != 0)
                    n_flags += 1
    return n_iou, n_flags


def same_eval(got, ev):
    for name in ("precision", "recall"):
        a, b = got.eval[name], ev.eval[name]
        assert a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64)), name
    assert list(got.results) == list(ev.results)
    for k in ev.results:
        assert np.float64(got.results[k]).view(np.uint64) == \
            np.float64(ev.results[k]).view(np.uint64), k
    with redirect_stdout(io.StringIO()) as out:
        got.print_results()
    assert out.getvalue() == ev.printed


EVALUATORS = {"segm": CaptureSegm, "bbox": CaptureBbox}


@pytest.mark.parametrize("iou_type", ["segm", "bbox"])
@pytest.mark.parametrize("max_dets", [300, 40])
def test_add_batch_equals_oracle(cuda_device, iou_type, max_dets):
    batches, images = stream(100)
    got = EVALUATORS[iou_type](CATS, images, max_dets=max_dets)
    for ids, items, anns, _, _ in batches:
        got.add_batch(items, ids, anns, category_ids=CMAP)
    got.run()
    gts, dts, gmap, dmap = oracle_inputs(batches, iou_type)
    ev = run_oracle(gts, dts, images, iou_type, max_dets)
    assert got.params.img_ids == ev.params.img_ids and got.params.cat_ids == ev.params.cat_ids
    n_iou, n_flags = check_pairs(ev, got, gmap, dmap)
    assert n_iou > 500 and n_flags > 300
    same_eval(got, ev)
    assert (ev.eval["precision"] > 0).any()
    assert max(sum(d["image_id"] == i for d in dts) for i in ev.params.img_ids) == 300
    flags = np.concatenate([e["dt_ignore"].ravel() for e in ev.eval_imgs if e is not None])
    assert flags.any() and not flags.all()


def records(e):
    return [np.concatenate([x[i] for x in parts]) for parts in (e._dets, e._gts)
            for i in range(len(parts[0]))]


@pytest.mark.parametrize("iou_type", ["segm", "bbox"])
def test_add_results_equals_add_batch_and_oracle(cuda_device, iou_type):
    batches, images = stream(200)
    a = EVALUATORS[iou_type](CATS, images, max_dets=60)
    b = EVALUATORS[iou_type](CATS, images, max_dets=60)
    for ids, items, anns, _, _ in batches:
        a.add_batch(items, ids, anns, category_ids=CMAP)
        b.add_results(api_utils.unmold_coco_results_batch(items, ids, category_ids=CMAP), anns,
                      ids)
    for x, y in zip(records(a), records(b)):
        assert x.dtype == y.dtype and np.array_equal(x, y)
    b.run()
    gts, dts, gmap, dmap = oracle_inputs(batches, iou_type)
    ev = run_oracle(gts, dts, images, iou_type, 60)
    n_iou, n_flags = check_pairs(ev, b, gmap, dmap)
    assert n_iou > 500 and n_flags > 300
    same_eval(b, ev)


def test_lvis_and_coco_evaluators_in_one_unmold(cuda_device):
    batches, images = stream(300)
    make = lambda: [evaluate.COCOevalSegm(polygons=True), CaptureSegm(CATS, images),  # noqa: E731
                    evaluate.COCOevalBbox(), CaptureBbox(CATS, images, max_dets=50)]
    together, apart = make(), make()
    for ids, items, anns, _, _ in batches:
        api_utils.unmold_coco_eval_batch(items, ids, anns, together, category_ids=CMAP)
        for e in apart:
            e.add_batch(items, ids, anns, category_ids=CMAP)
    for x, y in zip(together, apart):
        for r, s in zip(records(x), records(y)):
            assert np.array_equal(r, s)
        x.accumulate()
        y.accumulate()
        for name in ("precision", "recall"):
            assert np.array_equal(x.eval[name].view(np.uint64), y.eval[name].view(np.uint64))
        assert (x.eval["precision"] > 0).any()


def test_cross_check_equals_cocoevalsegm(cuda_device):
    """No crowds, every category without ground truth listed as negative, nothing not exhaustive,
    at most 100 detections per image: LVISEvalSegm is COCOevalSegm at maxDets 100."""
    batches, images = stream(400, [([1, 2], [(160, 200), (120, 96)], 100, 100),
                                   ([3], [(97, 203)], 80, 100)], cross_check=True)
    cat_ids = [c["id"] for c in CATS]
    lvis = evaluate.LVISEvalSegm(CATS, images)
    coco = evaluate.COCOevalSegm(cat_ids=cat_ids, polygons=True)
    for ids, items, anns, _, _ in batches:
        api_utils.unmold_coco_eval_batch(items, ids, anns, [lvis, coco], category_ids=CMAP)
    lvis.accumulate()
    coco.accumulate()
    for name in ("precision", "recall"):
        want = np.ascontiguousarray(coco.eval[name][..., -1])
        assert np.array_equal(lvis.eval[name].view(np.uint64), want.view(np.uint64)), name
    assert (lvis.eval["precision"] > 0).any()
