"""Boundary IoU evaluation on the device (mrx_mask_boundary / mrx_coco_boundary_ious and
evaluate.COCOevalBoundary): boundary planes bit for bit against boundary_iou_api's mask_to_boundary
on the real cv2 (tests/boundary_cocoeval_oracle.py), for ground truth over the whole image and for
predictions inside their boxes; then IoUs bit for bit, match and ignore flags, and the accumulated
arrays and stats exactly equal to the restated COCOeval for "boundary"; and one unmold feeding a
segm, a bbox and a boundary evaluator as three separate add_batch calls would."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest

import boundary_cocoeval_oracle as bo
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate, synth
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import MaskBatch, UnmoldEngine

from helpers import item_of, prepared_engine
from test_gpu_cocoeval import check_pairs, oracle_inputs, rle_of, same_eval

pytestmark = pytest.mark.gpu


class Capture(evaluate.COCOevalBoundary):
    """Keeps every batch's device results for the per-pair checks."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.batches = []

    def _record(self, image_ids, res, *rest):
        self.batches.append((list(image_ids), res))
        super()._record(image_ids, res, *rest)


def unpacked(planes, geom, b, k):
    H, W = int(geom[b, 0]), int(geom[b, 1])
    wb = (W + 7) // 8
    o = int(planes.d_packed_off[b].item()) + k * H * wb
    return np.unpackbits(planes.d_packed[o:o + H * wb].cpu().numpy().reshape(H, wb),
                         axis=1)[:, :W].astype(bool)


# ----------------------------------------------------------------------------- boundary planes
def _gt_masks(rng, H, W, M):
    ms = []
    for k in range(M):
        m = np.zeros((H, W), bool)
        if k == 0:
            m[:] = True                                         # the full image
        elif k == 1:
            pass                                                # empty
        elif k == 2:                                            # touching all four edges
            m[:, :max(W // 3, 1)] = True
            m[:max(H // 3, 1), :] = True
            m[-1, :] = True
            m[:, -1] = True
        else:
            y1, x1 = rng.integers(0, H), rng.integers(0, W)
            m[y1:y1 + rng.integers(1, H + 1), x1:x1 + rng.integers(1, W + 1)] = True
            m &= rng.random((H, W)) < rng.choice([1.0, 0.97, 0.6])
        ms.append(m)
    return np.stack(ms, axis=2)


SHAPES = [(1, 1), (37, 5), (5, 37), (16, 24), (9, 64), (800, 1333), (1024, 1024), (61, 203)]


@pytest.mark.parametrize("ratio", [0.005, 0.02, 0.5])
def test_ground_truth_boundaries_equal_cv2(cuda_device, ratio):
    rng = np.random.default_rng(int(ratio * 1000))
    geoms = [[H, W, H, W, 0, 0, H, W] for H, W in SHAPES]
    masks = [_gt_masks(rng, H, W, 7) for H, W in SHAPES]
    gt = MaskBatch(N.load(), cuda_device, geoms, [np.zeros(7, np.int32)] * len(SHAPES), masks)
    bp = gt.boundary_planes(ratio)
    areas = bp.d_areas.cpu().numpy()
    assert np.array_equal(bp.d_extents.cpu().numpy(), gt.planes.d_extents.cpu().numpy())
    n_kept_mask = 0
    for b, (H, W) in enumerate(SHAPES):
        for k in range(7):
            want = bo.mask_to_boundary(masks[b][:, :, k], ratio).astype(bool)
            got = unpacked(bp, gt.geom, b, k)
            assert np.array_equal(got, want), (H, W, k, ratio)
            assert areas[b, k] == want.sum()
            n_kept_mask += bool(want.sum()) and np.array_equal(want, masks[b][:, :, k])
    assert n_kept_mask > 0           # d above a side somewhere: the boundary is the mask


@pytest.mark.parametrize("ratio", [0.005, 0.02, 0.5])
def test_prediction_boundaries_equal_cv2(cuda_device, ratio):
    rng = np.random.default_rng(7 + int(ratio * 100))
    shapes = [(800, 1333), (75, 333), (17, 9), (1024, 1024)]
    ims = [synth.make_image(rng, hw, 30, num_classes=4, max_instances=32,
                            **({} if min(hw) > 64 else dict(min_box=1, max_box_frac=1.0)))
           for hw in shapes]
    ref = api_utils.unmold_detections_batch([item_of(im, np.float32) for im in ims])
    eng = prepared_engine(ims, 32, 4, np.float32)
    eng.enqueue_expand_packed()
    bp = eng.boundary_planes(ratio)
    areas, ext = bp.d_areas.cpu().numpy(), bp.d_extents.cpu().numpy()
    n = 0
    for b, (boxes, _, _, masks) in enumerate(ref):
        for k in range(masks.shape[2]):
            m = masks[:, :, k]
            want = bo.mask_to_boundary(m, ratio).astype(bool)
            # only the bytes that hold a pixel of the box are written: compare inside the box
            y1, x1 = max(int(boxes[k, 0]), 0), max(int(boxes[k, 1]), 0)
            y2, x2 = min(int(boxes[k, 2]), m.shape[0]), min(int(boxes[k, 3]), m.shape[1])
            inside = np.zeros(m.shape, bool)
            inside[y1:y2, x1:x2] = True
            assert not (want & ~inside).any()
            got = unpacked(bp, eng.layout.geom, b, k)
            assert np.array_equal(got[y1:y2, x1:x2], want[y1:y2, x1:x2]), (b, k, ratio)
            assert areas[b, k] == want.sum()
            ys, xs = np.nonzero(m)          # the boundary's extents are the mask's
            box = [ys.min(), xs.min(), ys.max() + 1, xs.max() + 1] if ys.size else [0, 0, 0, 0]
            assert ext[b, k].tolist() == box, (b, k)
            n += 1
    assert n > 40


# ----------------------------------------------------------------------------- evaluator
def make_batch(seed, shapes, n, R, classes):
    """items, annotation lists (RLE ground truth with crowds, an empty mask per image, some without
    `area`), the ground-truth masks and the unmolded predictions of one batch."""
    rng = np.random.default_rng(seed)
    ims = [synth.make_image(rng, hw, n, num_classes=classes, max_instances=R,
                            **({} if min(hw) > 64 else dict(min_box=1, max_box_frac=1.0)))
           for hw in shapes]
    for im in ims:       # equal scores within an image and across images
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
                del ann["area"]
            a.append(ann)
            ms.append(masks[:, :, k])
        H, W = masks.shape[:2]
        a.append({"category_id": int(cls[0]) if cls.size else 1, "iscrowd": 0, "area": 50.0,
                  "segmentation": rle_of(np.zeros((H, W), bool))})
        ms.append(np.zeros((H, W), bool))
        anns.append(a)
        gt_masks.append(ms)
    preds = api_utils.unmold_detections_batch(items)
    return items, anns, gt_masks, preds


STREAM = [  # (image ids, shapes, n, R, classes)
    ([30, 10], [(17, 9), (75, 333)], 12, 16, 3),
    ([20, 5, 40], [(96, 128), (33, 100), (64, 64)], 40, 48, 3),
    ([7], [(800, 1333)], 60, 64, 4),
]


def stream_batches(seed):
    return [(ids,) + make_batch(seed + s, shapes, n, R, classes)
            for s, (ids, shapes, n, R, classes) in enumerate(STREAM)]


def run_oracle(gts, dts, ratio, **params):
    p = bo.Params()
    for k, v in params.items():
        setattr(p, k, v)
    ev = bo.COCOevalBoundaryOracle(gts, dts, p, ratio)
    ev.evaluate()
    ev.accumulate()
    with redirect_stdout(io.StringIO()) as out:
        ev.summarize()
    ev.printed = out.getvalue()
    return ev


@pytest.mark.parametrize("ratio,params", [
    (0.02, dict()),
    (0.005, dict(iouThrs=np.array([0.3, 0.5, 0.75, 1.0]), maxDets=[1, 5, 20])),
    (0.1, dict(areaRng=[[0, 1e10], [0, 100], [100, 2000], [2000, 1e10], [1024, 9216]],
               areaRngLbl=["all", "small", "medium", "large", "mid"], maxDets=[2, 10, 20])),
])
def test_add_batch_equals_oracle(cuda_device, ratio, params):
    batches = stream_batches(900)
    kw = {"iou_thrs": params.get("iouThrs"), "max_dets": params.get("maxDets", (1, 10, 100)),
          "area_rng": params.get("areaRng"), "area_rng_lbl": params.get("areaRngLbl")}
    got = Capture(dilation_ratio=ratio, **kw)
    for ids, items, anns, _, _ in batches:
        got.add_batch(items, ids, anns)
    got.evaluate()
    got.accumulate()
    gts, dts, gmap, dmap = oracle_inputs(batches)
    ev = run_oracle(gts, dts, ratio, **params)
    assert got.params.imgIds == ev.params.imgIds and got.params.catIds == ev.params.catIds
    n_iou, n_flags = check_pairs(ev, got, gmap, dmap)
    assert n_iou > 500 and n_flags > 500
    same_eval(got, ev)
    assert (ev.eval["precision"] > 0).any() and any(g["iscrowd"] for g in gts)
    # the boundary decides some pairs: their IoU is below the mask IoU
    p = bo.Params()
    for k, v in params.items():
        setattr(p, k, v)
    seg = bo.COCOevalOracle(gts, dts, p)
    seg.evaluate()
    lower = sum(int((ev.ious[key] < seg.ious[key]).sum()) for key in ev.ious if len(ev.ious[key]))
    if ratio <= 0.02:        # (at 0.1 every synthetic object is all boundary)
        assert lower > 50


def test_add_results_equals_add_batch(cuda_device):
    cmap = [10 * c + 3 for c in range(4)]
    a = evaluate.COCOevalBoundary(max_dets=(1, 5, 20))
    b = evaluate.COCOevalBoundary(max_dets=(1, 5, 20))
    for ids, items, anns, _, _ in stream_batches(950):
        for a_ in anns:
            for ann in a_:
                ann["category_id"] = cmap[ann["category_id"]]
        a.add_batch(items, ids, anns, category_ids=cmap)
        b.add_results(api_utils.unmold_coco_results_batch(items, ids, category_ids=cmap), anns,
                      ids)
    for e in (a, b):
        e.accumulate()
    for name in ("precision", "recall", "scores"):
        assert np.array_equal(a.eval[name].view(np.uint64), b.eval[name].view(np.uint64)), name
    assert (a.eval["precision"] > 0).any()


def test_polygon_ground_truth(cuda_device):
    """Polygon ground truth (polygons=True) scores as its rasterised RLE does."""
    rng = np.random.default_rng(77)
    ims = [synth.make_image(rng, (120, 160), 20, num_classes=3, max_instances=24),
           synth.make_image(rng, (97, 203), 20, num_classes=3, max_instances=24)]
    items = [item_of(im, np.float32) for im in ims]
    preds = api_utils.unmold_detections_batch(items)
    polys, rles = [], []
    for (boxes, cls, _, _), im in zip(preds, ims):
        H, W = im.original_image_shape[:2]
        p, r = [], []
        for k in range(cls.shape[0]):
            y1, x1, y2, x2 = (int(v) + int(s) for v, s in zip(boxes[k], rng.integers(-3, 4, 4)))
            poly = [float(x1), float(y1), float(x2), float(y1 + 2), float(x2 - 3), float(y2),
                    float(x1 + 1), float(y2 - 1)]
            ann = {"category_id": int(cls[k]), "iscrowd": 0, "area": 100.0, "id": k + 1}
            p.append(dict(ann, segmentation=[poly]))
            m = evaluate.ann_to_mask({"segmentation": [poly]}, H, W).astype(bool)
            r.append(dict(ann, segmentation=rle_of(m)))
        polys.append(p)
        rles.append(r)
    a = evaluate.COCOevalBoundary(polygons=True)
    b = evaluate.COCOevalBoundary()
    a.add_batch(items, [1, 2], polys)
    b.add_batch(items, [1, 2], rles)
    for e in (a, b):
        e.accumulate()
    for name in ("precision", "recall", "scores"):
        assert np.array_equal(a.eval[name].view(np.uint64), b.eval[name].view(np.uint64)), name
    assert (a.eval["recall"] > -1).any()


def test_one_unmold_for_three_evaluators(cuda_device, monkeypatch):
    from test_gpu_cocoeval_bbox import CMAP, make_batch as bbox_batch

    batches = [([1, 2], *bbox_batch(1000, [(75, 333), (96, 128)], 30, 32, 3, CMAP)),
               ([3], *bbox_batch(1001, [(800, 1333)], 60, 64, 3, CMAP))]
    kw = dict(max_dets=(1, 5, 20))

    def three():
        return [evaluate.COCOevalSegm(**kw), evaluate.COCOevalBbox(**kw),
                evaluate.COCOevalBoundary(**kw)]

    together, apart = three(), three()
    for ids, items, anns in batches:
        for e in apart:
            e.add_batch(items, ids, anns, category_ids=CMAP)
    prepares = []
    prepare = UnmoldEngine.enqueue
    monkeypatch.setattr(UnmoldEngine, "enqueue",
                        lambda self, *a, **kw: (prepares.append(1), prepare(self, *a, **kw))[1])
    for ids, items, anns in batches:
        api_utils.unmold_coco_eval_batch(items, ids, anns, together, category_ids=CMAP)
    assert len(prepares) == len(batches)
    for a, b in zip(together, apart):
        for e in (a, b):
            e.accumulate()
            with redirect_stdout(io.StringIO()):
                e.summarize()
        for name in ("precision", "recall", "scores"):
            assert np.array_equal(a.eval[name].view(np.uint64), b.eval[name].view(np.uint64))
        assert np.array_equal(a.stats.view(np.uint64), b.stats.view(np.uint64))
    assert not np.array_equal(together[1].stats, together[2].stats)
