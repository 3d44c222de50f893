"""COCO polygon ground truth rasterised on the device (mrx_poly_decode, then mrx_mask_extents):
the planes must equal np.packbits of the polygon oracle's masks bit for bit, the areas and extents
the oracle's; mixed batches must equal per-kind ones; and unmold_compute_ap_batch,
COCOevalSegm(polygons=True) and ann_to_mask must give what the same annotations give as RLE."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest

import coco_oracle as co
import cocoeval_oracle as ceo
import polygon_oracle as po
from bbox_oracle import extract_bboxes
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate, synth
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import BatchLayout, MaskBatch

from helpers import item_of

pytestmark = pytest.mark.gpu


def _geom(H, W):
    return [H, W, H, W, 0, 0, H, W]


def _quantise(xy, step):
    return [float(v) for v in (np.round(np.asarray(xy) / step) * step if step else xy)]


def _part(rng, H, W, kind, step):
    """One polygon part of `kind` in (or around) an H x W image, coordinates on a grid of `step`
    (0: any real)."""
    cy, cx = rng.uniform(-0.2, 1.2) * H, rng.uniform(-0.2, 1.2) * W
    r = rng.uniform(0.1, 0.8) * max(H, W)
    if kind == "convex":
        t = np.sort(rng.uniform(0, 2 * np.pi, int(rng.integers(3, 12))))
        xy = np.stack([cx + r * np.cos(t), cy + r * np.sin(t)], 1)
    elif kind == "star":
        n = int(rng.integers(5, 12))
        t = np.linspace(0, 2 * np.pi, 2 * n, endpoint=False)
        rad = np.where(np.arange(2 * n) % 2, r * 0.4, r)
        xy = np.stack([cx + rad * np.cos(t), cy + rad * np.sin(t)], 1)
    elif kind == "self":           # random vertices: self-intersecting
        xy = np.stack([rng.uniform(-0.3, 1.3, 8) * W, rng.uniform(-0.3, 1.3, 8) * H], 1)
    elif kind == "collinear":
        a = rng.uniform(0, 1, 5)
        xy = np.stack([a * W, a * H], 1)
    else:                          # "degenerate": repeated vertices
        xy = np.repeat(np.stack([rng.uniform(0, W, 3), rng.uniform(0, H, 3)], 1), 2, axis=0)
    return _quantise(xy.ravel(), step)


def _instances(rng, H, W, n):
    """n polygon annotations: every kind and grid, 1-3 parts, with 1-2 point later parts."""
    kinds = ["convex", "star", "self", "collinear", "degenerate"]
    out = []
    for k in range(n):
        step = [0, 1, 0.5, 0.1][k % 4]
        parts = [_part(rng, H, W, kinds[k % len(kinds)], step)]
        for _ in range(int(rng.integers(0, 3))):
            parts.append(_part(rng, H, W, kinds[int(rng.integers(0, 3))], step))
        if k % 6 == 5:
            parts.append(_quantise(rng.uniform(0, 1, 2) * [W, H], step))    # one vertex
        if k % 6 == 4:
            parts.append(_quantise(rng.uniform(0, 1, 5) * [W, H, W, H, W], step))  # odd length
        out.append(parts)
    return out


def _from_coco(geoms, segms, class_ids=None):
    """MaskBatch.from_coco on the current device; (batch, [planes [M_b, H_b, wb] per image],
    areas, extents)."""
    import torch

    dev = torch.device("cuda", torch.cuda.current_device())
    if class_ids is None:
        class_ids = [np.ones(len(s), np.int32) for s in segms]
    gt = MaskBatch.from_coco(N.load(), dev, geoms, class_ids, segms)
    layout = BatchLayout(gt.geom, gt.R, limits=False)
    packed = gt.planes.d_packed.cpu().numpy()
    planes = []
    for b in range(gt.n):
        lo, hi = layout.packed_span(b, gt.counts[b])
        planes.append(packed[lo:hi].reshape(layout.packed_shape(b, gt.counts[b])))
    return gt, planes, gt.planes.d_areas.cpu().numpy(), gt.planes.d_extents.cpu().numpy()


def _oracle_masks(segms, H, W):
    return np.stack([po.ann_to_mask(s, H, W) if isinstance(s, list)
                     else po.decode(s["counts"] if isinstance(s["counts"], list)
                                    else co.rle_from_string(s["counts"]), H, W)
                     for s in segms], axis=2) if segms else np.zeros((H, W, 0), bool)


def _check(shapes_segms):
    geoms = [_geom(H, W) for (H, W), _ in shapes_segms]
    gt, planes, areas, ext = _from_coco(geoms, [s for _, s in shapes_segms])
    for b, ((H, W), segms) in enumerate(shapes_segms):
        m = _oracle_masks(segms, H, W)
        M = m.shape[2]
        want = np.packbits(m.transpose(2, 0, 1), axis=-1)
        for k in range(M):
            assert np.array_equal(planes[b][k], want[k]), (b, k, (H, W), segms[k])
        assert np.array_equal(areas[b, :M], m.sum((0, 1))), b
        assert np.array_equal(ext[b, :M], extract_bboxes(m)), b
        assert np.array_equal(gt.extents[b, :M], extract_bboxes(m)), b
    return gt


@pytest.mark.parametrize("hw", [(1, 1), (7, 13), (45, 1), (1, 37), (33, 65), (100, 37),
                                (64, 257), (480, 640)])
def test_random_polygons_equal_oracle(cuda_device, hw):
    """Convex, star, self-intersecting, collinear and degenerate parts, several parts per
    instance, vertices outside every side, real / integer / half / 0.1-step coordinates."""
    rng = np.random.default_rng(hw[0] * 1000 + hw[1])
    H, W = hw
    n = 24 if H * W < 100000 else 10
    _check([(hw, _instances(rng, H, W, n)), ((H + 3, W + 1), _instances(rng, H + 3, W + 1, 5))])


def test_known_answers(cuda_device):
    """The hand-worked annotations of the oracle's tests, through the device."""
    gt = _check([((20, 20), [[[0, 0, 10, 0, 10, 10, 0, 10]],                # the 10 x 10 square
                             [[0, 0, 1, 1, 2, 0]],                           # empty triangle
                             [[-0.1, -0.1, 5, -0.1, 5, 5, -0.1, 5]],
                             [[2, 3, 4, 5], [10, 10, 3, 2]],                 # a box list
                             [[0, 0, 10, 0, 10, 10, 0, 10], [5, 5, 15, 5, 15, 15, 5, 15]],
                             [[3, 0, 3, 40, 6, 40, 6, 0]]])])                # rows past H
    assert gt.planes.d_areas.cpu().numpy()[0, 0] == 100


def test_large_coordinates(cuda_device):
    """Vertices at +-1e5 and +-1e6: edges of millions of walked points, most outside the image."""
    _check([((40, 50), [[[-1e6, 5, 10, 1e6, 20.5, 3]],
                        [[1e5, -1e5, 30, 20, -1e5, 1e5]],
                        [[25, 20, 1e5, 21, 25, 22, -1e5, 23.3]]])])


def test_4k_image(cuda_device):
    rng = np.random.default_rng(7)
    _check([((2160, 3840), _instances(rng, 2160, 3840, 3))])


def test_mixed_batches_equal_per_kind(cuda_device):
    """Polygons next to compressed and uncompressed RLE in one batch give the planes that
    per-kind batches give; every RLE is the oracle's run list of a polygon."""
    rng = np.random.default_rng(11)
    shapes = [(60, 75), (33, 20)]
    polys = [_instances(rng, H, W, 9) for H, W in shapes]
    rles = [[{"size": [H, W], "counts": po.ann_to_rle(s, H, W)} for s in p]
            for (H, W), p in zip(shapes, polys)]
    mixed = []
    for p, r in zip(polys, rles):
        mixed.append([p[k] if k % 3 == 0 else
                      r[k] if k % 3 == 1 else
                      {"size": r[k]["size"], "counts": co.rle_to_string(r[k]["counts"])}
                      for k in range(len(p))])
    geoms = [_geom(H, W) for H, W in shapes]
    _, want, a_want, e_want = _from_coco(geoms, polys)
    for segms in (mixed, rles):
        _, got, a_got, e_got = _from_coco(geoms, segms)
        for b in range(2):
            assert np.array_equal(got[b], want[b])
        assert np.array_equal(a_got, a_want) and np.array_equal(e_got, e_want)
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    got = MaskBatch.from_rle(N.load(), dev, geoms, [np.ones(9, np.int32)] * 2, rles)
    assert np.array_equal(got.planes.d_areas.cpu().numpy(), a_want)


def test_mixed_batch_rle_errors_still_raise(cuda_device):
    """A malformed RLE next to polygons still raises, naming its instance."""
    segms = [[[[0, 0, 10, 0, 10, 10]], {"size": [20, 20], "counts": [3, 12]}]]
    with pytest.raises(ValueError, match=r"image 0, instance 1: the counts do not sum"):
        _from_coco([_geom(20, 20)], segms)


def test_ann_to_mask(cuda_device):
    rng = np.random.default_rng(5)
    for segm in _instances(rng, 41, 50, 6):
        got = evaluate.ann_to_mask({"segmentation": segm}, 41, 50)
        assert got.dtype == np.uint8 and got.shape == (41, 50)
        assert np.array_equal(got, po.ann_to_mask(segm, 41, 50).astype(np.uint8))
    rle = {"size": [41, 50], "counts": [7, 30, 2013]}
    assert np.array_equal(evaluate.ann_to_mask({"segmentation": rle}, 41, 50),
                          po.decode(rle["counts"], 41, 50).astype(np.uint8))


def test_compute_ap_polygons_equal_rle(cuda_device):
    """unmold_compute_ap_batch with polygon ground truth (with and without boxes) gives what the
    same ground truth as the oracle's RLE strings gives."""
    rng = np.random.default_rng(21)
    shapes = [(120, 200), (96, 128)]
    ims = [synth.make_image(rng, hw, 12, num_classes=4, max_instances=16) for hw in shapes]
    items = [item_of(im, np.float32) for im in ims]
    gts_p, gts_r = [], []
    for im, (H, W) in zip(ims, shapes):
        polys = _instances(rng, H, W, 8)
        cls = rng.integers(1, 4, 8).astype(np.int32)
        masks = _oracle_masks(polys, H, W)
        rles = [{"size": [H, W], "counts": co.rle_to_string(po.ann_to_rle(s, H, W))} for s in polys]
        gts_p.append((extract_bboxes(masks), cls, polys))
        gts_r.append((extract_bboxes(masks), cls, rles))
    thr = np.arange(0.5, 1.0, 0.05)
    for boxes in (True, False):
        gp = [(b if boxes else None, c, s) for b, c, s in gts_p]
        gr = [(b if boxes else None, c, s) for b, c, s in gts_r]
        got = api_utils.unmold_compute_ap_batch(items, gp, thr)
        want = api_utils.unmold_compute_ap_batch(items, gr, thr)
        for g, w in zip(got, want):
            assert set(g) == set(w)
            for key in w:
                assert g[key].dtype == w[key].dtype, key
                assert np.array_equal(g[key], w[key], equal_nan=True), key


def _cocoeval_inputs(seed):
    """Three images of polygon annotations plus crowd RLE, detections as RLE of other polygons."""
    rng = np.random.default_rng(seed)
    shapes = [(60, 80), (97, 45), (33, 120)]
    ids = [3, 1, 2]
    anns_p, anns_r, results, gts, dts = [], [], [], [], []
    for img, (H, W) in zip(ids, shapes):
        polys = _instances(rng, H, W, 10)
        ap, ar = [], []
        for k, s in enumerate(polys):
            m = po.ann_to_mask(s, H, W)
            cat = int(rng.integers(1, 4))
            crowd = k % 5 == 4
            rle = {"size": [H, W], "counts": co.rle_to_string(po.ann_to_rle(s, H, W))}
            area = float(m.sum()) + (0.5 if k % 2 else 0.0)
            ap.append({"category_id": cat, "segmentation": rle if crowd else s,
                       "iscrowd": int(crowd), "area": area, "id": len(gts) + 1})
            ar.append(dict(ap[-1], segmentation=rle))
            gts.append({"image_id": img, "category_id": cat, "mask": m, "iscrowd": int(crowd),
                        "area": area})
        for s in _instances(rng, H, W, 12):
            m = po.ann_to_mask(s, H, W)
            cat, score = int(rng.integers(1, 4)), float(np.round(rng.uniform(), 1))
            results.append({"image_id": img, "category_id": cat, "score": score,
                            "segmentation": {"size": [H, W],
                                             "counts": co.rle_to_string(po.ann_to_rle(s, H, W))}})
            dts.append({"image_id": img, "category_id": cat, "mask": m, "score": score})
        anns_p.append(ap)
        anns_r.append(ar)
    return ids, shapes, anns_p, anns_r, results, gts, dts


def test_cocoeval_polygons_equal_rle_and_oracle(cuda_device):
    ids, shapes, anns_p, anns_r, results, gts, dts = _cocoeval_inputs(31)
    got = evaluate.COCOevalSegm(polygons=True)
    got.add_results(results, anns_p, ids, image_shapes=shapes)
    rle = evaluate.COCOevalSegm()
    rle.add_results(results, anns_r, ids)
    for ev in (got, rle):
        ev.evaluate()
        ev.accumulate()
        with redirect_stdout(io.StringIO()):
            ev.summarize()
    oracle = ceo.COCOevalOracle(gts, dts, ceo.Params())
    oracle.evaluate()
    oracle.accumulate()
    with redirect_stdout(io.StringIO()):
        oracle.summarize()
    for name in ("precision", "recall", "scores"):
        for other in (rle.eval, oracle.eval):
            assert np.array_equal(got.eval[name].view(np.uint64), other[name].view(np.uint64)), name
    assert np.array_equal(got.stats, rle.stats) and np.array_equal(got.stats, oracle.stats)
    # polygon-only ground truth and no detections: the shape must be given
    ev = evaluate.COCOevalSegm(polygons=True)
    with pytest.raises(ValueError, match="image 9: its ground truth is polygons only"):
        ev.add_results([], [[a for a in anns_p[0] if not a["iscrowd"]]], [9])
