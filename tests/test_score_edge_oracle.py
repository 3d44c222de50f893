"""CPU checks of the scoring-edge inputs (tests/score_edge_inputs.py) and of the reference loops
test_gpu_score_edges.py holds the kernels to: each builder really produces the ties and bounds it
is named for (counted, so an edit cannot drop one silently), and each variant of the references
-- a model of one mutant in tools/mutate_eval.py -- changes the expected output on the GPU
test's own inputs."""
import numpy as np
import pytest

import bbox_cocoeval_oracle as bo
import cocoeval_oracle as co
import eval_oracle as eo
import lvis_oracle as lo
import score_edge_inputs as se
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N


def test_limits_are_the_headers():
    assert se.MAX_T == N.MRX_MAX_IOU_THRESHOLDS and se.MAX_A == N.MRX_MAX_AREA_RANGES
    assert len(se.thresholds64()) == se.MAX_T and len(se.area_ranges16()) == se.MAX_A


def test_every_default_threshold_is_a_small_quotient():
    """Every COCO threshold but 0.8999999999999999 is i / u for a union u <= 20."""
    exact = [t for t in co.Params().iouThrs
             if any(i / u == t for u in range(1, 21) for i in range(u + 1))]
    assert len(exact) == 9 and 0.8999999999999999 not in exact
    assert 0.8999999999999999 in co.Params().iouThrs


@pytest.fixture(scope="module")
def match_case():
    return se.coco_match_case(11)


def test_coco_match_case_holds_its_edges(match_case):
    c = match_case
    thr = c["thresholds"]
    kept = [(b, i) for b in range(c["B"]) for i in range(c["pred_counts"][b])
            if c["pred_keep"][b, i]]
    same = np.concatenate([c["iou"][b, i, :c["gt_counts"][b]][
        c["gt_cat"][b, :c["gt_counts"][b]] == c["pred_cat"][b, i]] for b, i in kept])
    on = {t: int(np.sum(same == t)) for t in thr}
    assert sum(v > 0 for v in on.values()) >= 16, on        # IoUs exactly on many thresholds
    assert on[0.5] and on[se.CAP] and on[0.0]
    below = sum(int(np.sum(same == np.nextafter(t, 0))) for t in set(thr) if t > 0)
    above = sum(int(np.sum(same == np.nextafter(t, 1))) for t in set(thr) if t < se.CAP)
    assert below > 10 and above > 10
    assert np.sum(same == 1.0) > 0
    lane32 = [p for p in c["planted"] if p[3] - p[2] == 32]
    lane1 = [p for p in c["planted"] if p[3] - p[2] == 1]
    assert len(lane32) >= 5 and len(lane1) >= 20
    assert sorted(set(c["gt_counts"].tolist())) == [0, 1, 31, 32, 33, 64, 65]
    assert (c["pred_counts"] == 0).any() and (c["gt_counts"] == 0).any()
    assert (c["pred_keep"][c["pred_counts"] > 0] == 0).any()
    # categories interleaved within an image, a prediction category without ground truth
    assert any(len(set(c["gt_cat"][b, :4].tolist())) > 1 for b in range(c["B"]))
    assert (c["pred_cat"] == 3).any()
    # areas on and one ulp / one unit beside 32^2, 96^2 and the custom bounds, and 0
    for v in (1024.0, 9216.0, np.nextafter(1024.0, 0), np.nextafter(9216.0, np.inf), 0.0,
              1023.5, 1.0):
        assert (c["gt_area"] == v).any(), v
    for v in (1024, 1023, 1025, 9216, 9217, 0):
        assert (c["pred_area"] == v).any(), v
    f64 = se.coco_match_case(11, area_type=np.float64)
    assert (f64["pred_area"] == np.nextafter(1024.0, 0)).any()
    assert (c["gt_crowd"][c["gt_counts"].nonzero()[0]] == 1).any()


def test_coco_match_reference_meets_the_edges(match_case):
    """On the reference's own matches: a crowd matched by several detections, an ignored
    candidate above a matched non-ignored one, matches at the threshold exactly, matches of
    j >= 32, and ignore flags from both rules."""
    c = match_case
    match, ignore = se.expected_coco_match(c)
    A, T = len(c["area_rng"]), len(c["thresholds"])
    crowd_multi = above = at_thr = wide = 0
    for a in range(A):
        for t in range(T):
            for b in range(c["B"]):
                m = match[a, t, b]
                js, counts = np.unique(m[m >= 0], return_counts=True)
                crowd_multi += int(np.sum(c["gt_crowd"][b, js[counts > 1]]))
                wide += int(np.sum(m >= 32))
                for i in np.nonzero(m >= 0)[0]:
                    j = m[i]
                    v = c["iou"][b, i, j]
                    at_thr += v == c["thresholds"][t]
                    lo_, hi_ = c["area_rng"][a]
                    if not ignore[a, t, b, i]:
                        row = c["iou"][b, i, :c["gt_counts"][b]]
                        cat = c["gt_cat"][b, :c["gt_counts"][b]] == c["pred_cat"][b, i]
                        ig = c["gt_crowd"][b, :c["gt_counts"][b]].astype(bool) | \
                            (c["gt_area"][b, :c["gt_counts"][b]] < lo_) | \
                            (c["gt_area"][b, :c["gt_counts"][b]] > hi_)
                        above += int(np.any(cat & ig & (row > v)))
    assert crowd_multi > 10 and above > 10 and at_thr > 10 and wide > 10
    flags = ignore[ignore != 2]
    assert flags.any() and not flags.all()


def test_coco_match_cap_case():
    c = se.coco_match_cap_case()
    match, _ = se.expected_coco_match(c)
    assert match[0, 0, 0, 0] == 65533 and c["R2"] == 65534
    assert (match[:, :, 1] == -1).all()


@pytest.mark.parametrize("variant", co.MATCH_VARIANTS)
def test_coco_match_variants_change_the_expectation(match_case, variant):
    base = se.expected_coco_match(match_case)
    f64 = se.coco_match_case(11, area_type=np.float64)
    changed = [not all(np.array_equal(x, y) for x, y in
                       zip(se.expected_coco_match(c, variant), se.expected_coco_match(c)))
               for c in (match_case, f64)]
    assert all(changed), changed
    assert base[0].shape == (se.MAX_A, se.MAX_T, match_case["B"], match_case["R1"])


@pytest.fixture(scope="module")
def mask_case():
    return se.mask_match_case(12)


def test_mask_match_case_holds_its_edges(mask_case):
    c = mask_case
    ov = np.concatenate([c["overlaps"][b, :c["pred_counts"][b], :c["gt_counts"][b]].ravel()
                         for b in range(c["B"])])
    assert np.isnan(ov).sum() > 20
    for t in (0.5, 0.7, 0.75, 0.95, 0.55):
        assert (ov == np.float32(t)).sum() > 5, t
        assert (ov == np.nextafter(np.float32(t), np.float32(0))).sum() > 0 or \
            (ov == np.nextafter(np.float32(t), np.float32(1))).sum() > 0, t
    assert (ov == np.float32(c["score_threshold"])).sum() > 5
    s = c["scores"][c["pred_counts"] > 0]
    assert np.isnan(s).any() and len(np.unique(s[~np.isnan(s)])) < s.size / 2
    assert sum(p[3] - p[2] == 32 for p in c["planted"]) >= 5
    assert sum(p[3] - p[2] == 1 for p in c["planted"]) >= 20
    # float32(0.7) < 0.7: a NumPy 0.7 refuses it, a Python 0.7 (compared in float32) does not
    assert any(isinstance(t, float) for t in se.MASK_THRESHOLDS)
    assert any(isinstance(t, np.float64) for t in se.MASK_THRESHOLDS)
    assert (ov == np.float32(0.7)).sum() > 0 and np.float32(0.7) < np.float64(0.7)


@pytest.mark.parametrize("t", [0.7, 0.95])
def test_mask_match_python_and_numpy_thresholds_differ(mask_case, t):
    a = se.expected_mask_matches(mask_case, t, 0.0)
    b = se.expected_mask_matches(mask_case, np.float64(t), 0.0)
    assert not np.array_equal(a[1], b[1])


@pytest.mark.parametrize("variant", eo.MATCH_VARIANTS)
def test_mask_match_variants_change_the_expectation(mask_case, variant):
    c = mask_case
    changed = False
    for t in se.MASK_THRESHOLDS:
        want = se.expected_mask_matches(c, t, c["score_threshold"])
        got = se.expected_mask_matches(c, t, c["score_threshold"], variant)
        changed |= not all(np.array_equal(x, y) for x, y in zip(want, got))
    assert changed


@pytest.fixture(scope="module")
def planes():
    return se.planes_case(13)


def test_planes_hold_every_alignment(planes):
    wbs = [(im["W"] + 7) // 8 for im in planes]
    assert {w % 4 for w in wbs} == {0, 1, 2, 3}
    assert any(im["H"] * w % 2 for im, w in zip(planes, wbs))
    R = max(len(im["pred"]) for im in planes)
    buf, off = se.pack_slots(planes, "pred", R, 0)
    bases = {int(o + k * im["H"] * w) % 4 for o, im, w in zip(off, planes, wbs) for k in range(R)}
    assert bases == {0, 1, 2, 3}
    starts, ends, narrow, touch, last, empty = set(), set(), 0, 0, 0, 0
    for im in planes:
        for m1 in im["pred"]:
            for m2 in im["gt"]:
                a, b = se.extents(m1), se.extents(m2)
                if not (m1.any() and m2.any()):
                    empty += 1
                    continue
                y1, x1, y2, x2 = max(a[0], b[0]), max(a[1], b[1]), min(a[2], b[2]), min(a[3], b[3])
                if x2 > x1 and y2 > y1:
                    starts.add(x1 & 7)
                    ends.add((x2 - 1) & 7)
                    narrow += x2 - x1 == 1 or y2 - y1 == 1
                elif x2 == x1 and y2 > y1:
                    touch += 1
        last += sum(bool(m[-1, -1]) for m in im["pred"] + im["gt"])
        for m, q in zip(im["pred"] + im["gt"], im["pred_bnd"] + im["gt_bnd"]):
            y1, x1, y2, x2 = se.extents(m)
            assert not q.any() or (se.extents(q)[0] >= y1 and se.extents(q)[1] >= x1 and
                                   se.extents(q)[2] <= y2 and se.extents(q)[3] <= x2)
    assert starts == set(range(8)) and ends == set(range(8))
    assert narrow > 5 and touch > 0 and last > 3 and empty > 0


@pytest.mark.parametrize("variant", se.PAIR_VARIANTS)
def test_pair_variants_change_the_expectation(planes, variant):
    changed = 0
    for im in planes:
        for m1 in im["pred"]:
            for m2, crowd in zip(im["gt"], im["gt_crowd"]):
                i0, i1 = se.pair_counts(m1, m2), se.pair_counts(m1, m2, variant)
                a1, a2 = int(m1.sum()), int(m2.sum())
                changed += se.rle_iou_counts(i0, a1, a2, crowd) != \
                    se.rle_iou_counts(i1, a1, a2, crowd, variant)
    assert changed > 3


def test_box_dataset_lands_on_the_thresholds():
    ids, shapes, gts, dts = se.box_dataset()
    ev = bo.COCOevalBboxOracle([dict(g) for g in gts], [dict(d) for d in dts])
    ev.evaluate()
    ious = np.concatenate([np.ravel(v) for v in ev.ious.values() if len(v)])
    for t in co.Params().iouThrs:
        if t != 0.8999999999999999:
            assert (ious == t).any(), t
    assert (ious == 0).any() and (ious == 1).any()
    areas = {d["bbox"][2] * d["bbox"][3] for d in dts}
    assert {1024.0, 9216.0, 0.0, -12.0} <= areas
    assert any(1024.0 < a < 1024.001 for a in areas) and any(1023.9 < a < 1024.0 for a in areas)
    assert {1024.0, 9216.0, np.nextafter(1024.0, 0)} <= {g["area"] for g in gts}
    assert sum(g["image_id"] == 2 for g in gts) == 40
    assert not any(g["image_id"] == 3 for g in gts)
    # a crowd several detections match, in the reference's own evaluation
    e = [x for x in ev.evalImgs if x is not None and x["image_id"] == 5 and x["aRng"] == [0, 1e10]]
    crowd = [k for k, g in enumerate(gts) if g["iscrowd"] and g["image_id"] == 5]
    assert np.sum(e[0]["dtMatchIds"][0] == crowd[0]) >= 2


def test_box_union_contraction_changes_an_iou():
    """The fma mutant's union (da + g2 * g3 rounded once) changes a box IoU of the dataset."""
    _, _, gts, dts = se.box_dataset()
    diff = 0
    for d in dts:
        for g in gts:
            if g["image_id"] != d["image_id"] or g["iscrowd"]:
                continue
            D, G = d["bbox"], g["bbox"]
            da = D[2] * D[3]
            w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
            h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
            if w <= 0 or h <= 0:
                continue
            i = w * h
            diff += i / (da + G[2] * G[3] - i) != i / (se.fma_union(da, G[2], G[3]) - i)
    assert diff > 0


def test_lvis_cut_by_category_changes_the_kept_set():
    """LVIS's per-image cut counts every category; a cut per (image, category) keeps others."""
    _, _, _, dts = se.box_dataset()
    a = {d["id"] for d in lo.limit_dets_per_image(dts, 5)}
    b = {d["id"] for d in lo.limit_dets_per_image(dts, 5, per_category=True)}
    assert a != b
