"""The scoring kernels at their ties and bounds (inputs: tests/score_edge_inputs.py), bit for bit
against the loops as pycocotools, lvis-api and Matterport write them:

- mrx_coco_match / mrx_coco_match_f64area through the C ABI on constructed IoU, walk, keep,
  category, crowd and area tables: match and ignore for every (area range, threshold) against
  evaluateImg's loop (cocoeval_oracle.match_image), at T = MRX_MAX_IOU_THRESHOLDS,
  A = MRX_MAX_AREA_RANGES, and at R2 = 65534;
- mrx_mask_matches on constructed float32 overlaps: order, pred_match and gt_match against
  compute_matches' loop (eval_oracle.match_loop), thresholds as Python floats and as NumPy
  scalars, a score threshold equal to IoUs of the matrix;
- mrx_mask_extents, mrx_mask_overlaps, mrx_coco_ious and mrx_coco_boundary_ious on planes packed
  in NumPy at every byte alignment, against exact counts;
- coco_box_evaluate_batch's IoUs and areas against bbIou, and COCOevalBbox, COCOevalSegm and
  LVISEvalBbox end to end against their oracles on one dataset of exact-threshold IoUs."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

import bbox_cocoeval_oracle as bo
import coco_oracle
import cocoeval_oracle as co
import lvis_oracle as lo
import score_edge_inputs as se
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import engine, evaluate

pytestmark = pytest.mark.gpu


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


# ----------------------------------------------------------------------------- matches
def run_coco_match(c, f64):
    lib = N.load()
    A, T, B, R1, R2 = len(c["area_rng"]), len(c["thresholds"]), c["B"], c["R1"], c["R2"]
    match = torch.full((A, T, B, R1), -2, dtype=torch.int32, device="cuda")
    ignore = torch.full((A, T, B, R1), 2, dtype=torch.uint8, device="cuda")
    area = c["pred_area"].astype(np.float64 if f64 else np.int64)
    name = "mrx_coco_match_f64area" if f64 else "mrx_coco_match"
    args = [dev(c[k]) for k in ("iou", "pred_counts", "pred_cat", "pred_keep", "walk")] + \
        [dev(area)] + [dev(c[k]) for k in ("gt_counts", "gt_cat", "gt_crowd", "gt_area")]
    N.check(getattr(lib, name)(
        *args, N.double_array(c["thresholds"]), T,
        N.double_array(np.ravel(c["area_rng"])), A, match, ignore, B, R1, R2,
        N.stream_ptr(None)), name)
    return match.cpu().numpy(), ignore.cpu().numpy()


@pytest.mark.parametrize("seed,area_type", [(11, np.int64), (11, np.float64), (21, np.int64),
                                            (22, np.float64)])
def test_coco_match_equals_the_loop(cuda_device, seed, area_type):
    c = se.coco_match_case(seed, area_type=area_type)
    want_m, want_i = se.expected_coco_match(c)
    got_m, got_i = run_coco_match(c, area_type == np.float64)
    assert np.array_equal(got_m, want_m), np.argwhere(got_m != want_m)[:5]
    assert np.array_equal(got_i, want_i), np.argwhere(got_i != want_i)[:5]
    assert (want_m >= 0).sum() > 1000


@pytest.mark.parametrize("area_type", [np.int64, np.float64])
def test_coco_match_at_the_instance_cap(cuda_device, area_type):
    c = se.coco_match_cap_case(area_type)
    want_m, want_i = se.expected_coco_match(c)
    got_m, got_i = run_coco_match(c, area_type == np.float64)
    assert got_m[0, 0, 0, 0] == 65533
    assert np.array_equal(got_m, want_m) and np.array_equal(got_i, want_i)


def run_mask_matches(c, thresholds, score_threshold):
    lib = N.load()
    B, R1, R2, T = c["B"], c["R1"], c["R2"], len(thresholds)
    order = torch.full((B, R1), -2, dtype=torch.int32, device="cuda")
    pm = torch.full((T, B, R1), -2, dtype=torch.int32, device="cuda")
    gm = torch.full((T, B, R2), -2, dtype=torch.int32, device="cuda")
    args = [dev(c[k]) for k in ("overlaps", "pred_counts", "pred_cls", "scores")]
    N.check(lib.mrx_mask_matches(
        *args[:4], N.MRX_F32, dev(c["gt_counts"]), dev(c["gt_cls"]),
        N.double_array([engine.comparison_threshold(t) for t in thresholds]), T,
        engine.comparison_threshold(score_threshold), order, pm, gm, B, R1, R2,
        N.stream_ptr(None)), "mrx_mask_matches")
    return order.cpu().numpy(), pm.cpu().numpy(), gm.cpu().numpy()


@pytest.mark.parametrize("seed", [12, 31])
@pytest.mark.parametrize("score", ["zero", "on_an_iou", "on_an_iou_f64"])
def test_mask_matches_equal_the_loop(cuda_device, seed, score):
    c = se.mask_match_case(seed)
    sthr = {"zero": 0.0, "on_an_iou": c["score_threshold"],
            "on_an_iou_f64": np.float64(c["score_threshold"])}[score]
    thr = se.MASK_THRESHOLDS
    order, pm, gm = run_mask_matches(c, thr, sthr)
    matched = 0
    for t, th in enumerate(thr):
        w_order, w_pm, w_gm = se.expected_mask_matches(c, th, sthr)
        assert np.array_equal(order, w_order)
        assert np.array_equal(pm[t], w_pm), (th, np.argwhere(pm[t] != w_pm)[:5])
        assert np.array_equal(gm[t], w_gm), (th, np.argwhere(gm[t] != w_gm)[:5])
        matched += int((w_pm >= 0).sum())
    assert matched > 100


# ----------------------------------------------------------------------------- pair walk
def _side(imgs, key, R, lead, geom):
    buf, off = se.pack_slots(imgs, key, R, lead)
    counts = np.array([len(im[key]) for im in imgs], np.int32)
    regions = np.zeros((len(imgs), R, 4), np.int32)
    for b, im in enumerate(imgs):
        regions[b, :] = [0, 0, im["H"], im["W"]]
    return {"buf": dev(buf), "off": dev(off), "counts": dev(counts), "regions": dev(regions)}


def _extents(lib, s, geom, B, R):
    areas = torch.full((B, R), -1, dtype=torch.int64, device="cuda")
    ext = torch.full((B, R, 4), -1, dtype=torch.int32, device="cuda")
    N.check(lib.mrx_mask_extents(s["buf"], s["off"], s["counts"], geom, s["regions"], areas, ext,
                                 B, R, N.stream_ptr(None)), "mrx_mask_extents")
    s["areas"], s["ext"] = areas, ext
    return areas.cpu().numpy(), ext.cpu().numpy()


@pytest.mark.parametrize("lead", [0, 3])
def test_pair_walk_equals_exact_counts(cuda_device, lead):
    lib = N.load()
    imgs = se.planes_case(13 + lead)
    B = len(imgs)
    R1, R2 = max(len(im["pred"]) for im in imgs), max(len(im["gt"]) for im in imgs)
    geom = dev(np.array([[im["H"], im["W"], im["H"], im["W"], 0, 0, im["H"], im["W"]]
                         for im in imgs], np.int32))
    p = _side(imgs, "pred", R1, lead, geom)
    g = _side(imgs, "gt", R2, lead + 1, geom)
    q1 = _side(imgs, "pred_bnd", R1, lead, geom)
    q2 = _side(imgs, "gt_bnd", R2, lead + 1, geom)
    for s, key, R in ((p, "pred", R1), (g, "gt", R2), (q1, "pred_bnd", R1), (q2, "gt_bnd", R2)):
        areas, ext = _extents(lib, s, geom, B, R)
        for b, im in enumerate(imgs):
            for k, m in enumerate(im[key]):
                assert areas[b, k] == m.sum(), (key, b, k)
                if not key.endswith("bnd"):
                    assert tuple(ext[b, k]) == se.extents(m), (key, b, k)
    pred_cat = np.full((B, R1), -1, np.int32)
    keep = np.zeros((B, R1), np.uint8)
    gt_cat = np.full((B, R2), -1, np.int32)
    crowd = np.zeros((B, R2), np.uint8)
    for b, im in enumerate(imgs):
        pred_cat[b, :len(im["pred"])] = im["pred_cat"]
        keep[b, :len(im["pred"])] = im["pred_keep"]
        gt_cat[b, :len(im["gt"])] = im["gt_cat"]
        crowd[b, :len(im["gt"])] = im["gt_crowd"]
    st = N.stream_ptr(None)
    ov = torch.full((B, R1, R2), -7.0, dtype=torch.float32, device="cuda")
    N.check(lib.mrx_mask_overlaps(p["buf"], p["off"], p["counts"], p["areas"], p["ext"], R1,
                                  g["buf"], g["off"], g["counts"], g["areas"], g["ext"], R2,
                                  geom, ov, B, st), "mrx_mask_overlaps")
    d_cat, d_keep, d_gcat, d_crowd = dev(pred_cat), dev(keep), dev(gt_cat), dev(crowd)
    iou = torch.full((B, R1, R2), -7.0, dtype=torch.float64, device="cuda")
    N.check(lib.mrx_coco_ious(p["buf"], p["off"], p["counts"], p["areas"], p["ext"], d_cat,
                              d_keep, R1, g["buf"], g["off"], g["counts"], g["areas"], g["ext"],
                              d_gcat, d_crowd, R2, geom, iou, B, st), "mrx_coco_ious")
    biou = torch.full((B, R1, R2), -7.0, dtype=torch.float64, device="cuda")
    N.check(lib.mrx_coco_boundary_ious(
        p["buf"], p["off"], p["counts"], p["areas"], p["ext"], q1["buf"], q1["areas"], d_cat,
        d_keep, R1, g["buf"], g["off"], g["counts"], g["areas"], g["ext"], q2["buf"],
        q2["areas"], d_gcat, d_crowd, R2, geom, biou, B, st), "mrx_coco_boundary_ious")
    ov, iou, biou = ov.cpu().numpy(), iou.cpu().numpy(), biou.cpu().numpy()
    n_pairs = 0
    for b, im in enumerate(imgs):
        for i, (m1, b1) in enumerate(zip(im["pred"], im["pred_bnd"])):
            a1, ba1 = int(m1.sum()), int(b1.sum())
            for j, (m2, b2) in enumerate(zip(im["gt"], im["gt_bnd"])):
                a2, ba2 = int(m2.sum()), int(b2.sum())
                inter = se.pair_counts(m1, m2)
                want = se.f32_iou(inter, a1, a2)
                # 0 / 0 (both masks empty): NaN, whose sign and payload NumPy and CUDA spell
                # differently
                assert ov[b, i, j].view(np.uint32) == want.view(np.uint32) or \
                    np.isnan(ov[b, i, j]) and np.isnan(want) and a1 == a2 == 0, (b, i, j)
                if keep[b, i] and pred_cat[b, i] == gt_cat[b, j]:
                    cr = bool(crowd[b, j])
                    w = se.rle_iou_counts(inter, a1, a2, cr)
                    wb = min(w, se.rle_iou_counts(int(np.count_nonzero(b1 & b2)), ba1, ba2, cr))
                    n_pairs += inter > 0
                else:
                    w = wb = -7.0
                assert np.float64(iou[b, i, j]).view(np.uint64) == np.float64(w).view(np.uint64)
                assert np.float64(biou[b, i, j]).view(np.uint64) == \
                    np.float64(wb).view(np.uint64), (b, i, j)
    assert n_pairs > 100


# ----------------------------------------------------------------------------- boxes, end to end
CATS = [{"id": 7, "frequency": "f"}, {"id": 8, "frequency": "r"}]


def _anns(ids, gts, segm=False):
    out = []
    for img in ids:
        a = []
        for g in gts:
            if g["image_id"] == img:
                x = {"category_id": g["category_id"], "bbox": g["bbox"], "area": g["area"],
                     "iscrowd": g["iscrowd"]}
                if segm:
                    x["segmentation"] = coco_oracle.encode(g["mask"])
                a.append(x)
        out.append(a)
    return out


def _results(dts, segm=False):
    return [dict({"image_id": d["image_id"], "category_id": d["category_id"],
                  "score": d["score"], "bbox": d["bbox"]},
                 **({"segmentation": coco_oracle.encode(d["mask"])} if segm else {}))
            for d in dts]


def test_box_ious_and_areas_equal_bbiou(cuda_device):
    ids, _, gts, dts = se.box_dataset()
    R1 = max(sum(d["image_id"] == i for d in dts) for i in ids)
    R2 = max(sum(g["image_id"] == i for g in gts) for i in ids)
    n, cat = len(ids), {7: 0, 8: 1}
    pc, pcls = np.zeros(n, np.int32), np.full((n, R1), -1, np.int32)
    pb, ps = np.zeros((n, R1, 4)), np.zeros((n, R1))
    gc, gcat = np.zeros(n, np.int32), np.full((n, R2), -1, np.int32)
    gb, gcr, ga = np.zeros((n, R2, 4)), np.zeros((n, R2), np.uint8), np.zeros((n, R2))
    for b, img in enumerate(ids):
        for d in (d for d in dts if d["image_id"] == img):
            k = pc[b]
            pcls[b, k], pb[b, k], ps[b, k] = cat[d["category_id"]], d["bbox"], d["score"]
            pc[b] += 1
        for g in (g for g in gts if g["image_id"] == img):
            k = gc[b]
            gcat[b, k], gb[b, k], gcr[b, k], ga[b, k] = (cat[g["category_id"]], g["bbox"],
                                                         g["iscrowd"], g["area"])
            gc[b] += 1
    res = engine.coco_box_evaluate_batch(N.load(), pb, pc, pcls, ps, gc, gcat, gb, gcr, ga,
                                         np.arange(2, dtype=np.int32), co.Params())
    d_iou = res["d_iou"].cpu().numpy()
    checked = 0
    for b in range(n):
        for i in range(pc[b]):
            D = pb[b, i]
            assert np.float64(res["area"][b, i]).view(np.uint64) == \
                np.float64(D[2] * D[3]).view(np.uint64)
            for j in range(gc[b]):
                if gcat[b, j] != pcls[b, i]:
                    continue
                want = bo.bb_iou([D], [gb[b, j]], [gcr[b, j]])[0, 0]
                assert d_iou[b, i, j].view(np.uint64) == want.view(np.uint64), (b, i, j)
                checked += 1
    assert checked > 1500


def _same_coco(got, ev):
    for name in ("precision", "recall", "scores"):
        a, b = got.eval[name], ev.eval[name]
        assert a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64)), name
    with redirect_stdout(io.StringIO()) as x:
        got.summarize()
    with redirect_stdout(io.StringIO()) as y:
        ev.summarize()
    assert x.getvalue() == y.getvalue()
    assert (ev.eval["precision"] > 0).any()


def test_cocoeval_bbox_end_to_end(cuda_device):
    ids, _, gts, dts = se.box_dataset()
    got = evaluate.COCOevalBbox()
    got.add_results(_results(dts), _anns(ids, gts), ids)
    got.accumulate()
    ev = bo.COCOevalBboxOracle(gts, dts)
    ev.evaluate()
    ev.accumulate()
    _same_coco(got, ev)


def test_cocoeval_segm_end_to_end(cuda_device):
    ids, shapes, gts, dts = se.box_dataset()
    gts = [g for g in gts if g["mask"] is not None]
    dts = [d for d in dts if d["mask"] is not None]
    got = evaluate.COCOevalSegm()
    got.add_results(_results(dts, True), _anns(ids, gts, True), ids,
                    image_shapes=[shapes[i] for i in ids])
    got.accumulate()
    ev = co.COCOevalOracle(gts, dts)
    ev.evaluate()
    ev.accumulate()
    _same_coco(got, ev)


@pytest.mark.parametrize("max_dets", [300, 5])
def test_lvis_bbox_end_to_end(cuda_device, max_dets):
    ids, shapes, gts, dts = se.box_dataset()
    images = [{"id": i, "height": shapes[i][0], "width": shapes[i][1],
               "neg_category_ids": [7, 8] if i == 3 else [],
               "not_exhaustive_category_ids": [8] if i == 1 else []} for i in ids]
    got = evaluate.LVISEvalBbox(CATS, images, max_dets=max_dets)
    got.add_results(_results(dts), _anns(ids, gts), ids)
    got.run()
    p = lo.Params("bbox")
    p.max_dets = max_dets
    ev = lo.LVISEvalOracle(gts, dts, images, CATS, "bbox", p)
    ev.run()
    for name in ("precision", "recall"):
        a, b = got.eval[name], ev.eval[name]
        assert a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64)), name
    assert list(got.results) == list(ev.results)
    for k in ev.results:
        assert np.float64(got.results[k]).view(np.uint64) == \
            np.float64(ev.results[k]).view(np.uint64), k
    with redirect_stdout(io.StringIO()) as x:
        got.print_results()
    with redirect_stdout(io.StringIO()) as y:
        ev.print_results()
    assert x.getvalue() == y.getvalue()
