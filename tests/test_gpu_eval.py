"""Mask IoU, matches and AP against ground truth on the device (mrx_mask_extents / _overlaps /
_matches): everything must equal the restated upstream compute_overlaps_masks, compute_matches,
compute_ap and compute_ap_range (tests/eval_oracle.py) run on the masks unmold_detections_batch
returns -- overlaps bit for bit, NaN positions included."""
import io
from contextlib import redirect_stdout

import numpy as np
import pytest

import eval_oracle as eo
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate, synth

from helpers import item_of, prepared_engine

pytestmark = pytest.mark.gpu


def _same_f32(a, b):
    """Equal dtype and shape, NaN in the same places, every other value bit for bit."""
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb)
    assert np.array_equal(a[~na], b[~nb]) and np.array_equal(np.signbit(a[~na]), np.signbit(b[~nb]))


def _gt_of(ims, seed, dtype=np.float32, **kw):
    """Ground truth (boxes, class_ids, masks) per image: the unmolded jittered image."""
    rng = np.random.default_rng(seed)
    jit = [synth.jitter_ground_truth(im, rng, **kw) for im in ims]
    return [(b, c, m) for b, c, _, m in api_utils.unmold_detections_batch(
        [item_of(im, dtype) for im in jit])]


def _check(items, gts, thresholds=(0.5,), score_threshold=0.0, with_ap=True):
    got = api_utils.unmold_compute_ap_batch(items, gts, thresholds, score_threshold)
    ref = api_utils.unmold_detections_batch(items)
    assert len(got) == len(items)
    matched = 0
    for b, (g, (rb, rc, rs, rm)) in enumerate(zip(got, ref)):
        assert np.array_equal(g["rois"], rb) and np.array_equal(g["class_ids"], rc)
        assert np.array_equal(g["scores"], rs)
        assert g["pred_match"].shape == (len(thresholds), rb.shape[0])
        for t, thr in enumerate(thresholds):
            gm, pm, ov = eo.compute_matches(*gts[b], rb, rc, rs, rm, thr, score_threshold)
            if t == 0:
                _same_f32(g["overlaps"], ov)
            assert g["pred_match"][t].dtype == np.float64 and g["gt_match"][t].dtype == np.float64
            assert np.array_equal(g["pred_match"][t], pm), (b, thr)
            assert np.array_equal(g["gt_match"][t], gm), (b, thr)
            matched += int((pm > -1).sum())
            if with_ap and score_threshold == 0.0:
                ap = eo.compute_ap(*gts[b], rb, rc, rs, rm, thr)[0]
            else:
                ap = evaluate.ap_from_matches(pm, gm)[0]
            assert np.array_equal(g["ap"][t], ap, equal_nan=True), (b, thr, g["ap"][t], ap)
    return got, matched


@pytest.mark.parametrize("hw,n,R,kw", [
    ((96, 128), 12, 16, {}),
    ((75, 333), 37, 40, {}),
    ((17, 9), 3, 4, dict(min_box=1, max_box_frac=1.0)),
    ((33, 1000), 7, 8, {}),
])
def test_ap_equals_oracle_small_shapes(cuda_device, hw, n, R, kw):
    rng = np.random.default_rng(101)
    ims = [synth.make_image(rng, hw, n, num_classes=4, max_instances=R, **kw) for _ in range(3)]
    gts = _gt_of(ims, 102, max_shift=3, class_flip_frac=0.2)
    items = [item_of(im, np.float32) for im in ims]
    _check(items, gts, (0.5,))
    _check(items, gts, np.arange(0.5, 1.0, 0.05))
    _check(items, gts, [0.3, np.float64(0.6)], score_threshold=0.4)


def test_ap_full_size(cuda_device):
    """800x1333 with zero-area drops, and two configs[1] images: 100 predictions against 100
    jittered ground-truth instances, with real matches."""
    rng = np.random.default_rng(103)
    ims = [synth.make_image(rng, (800, 1333), 60, num_classes=81, max_instances=100,
                            zero_area_rows=(2, 30, 59)) for _ in range(2)]
    _, matched = _check([item_of(im, np.float64) for im in ims], _gt_of(ims, 104, np.float64))
    assert matched > 0
    ims = synth.make_batch(105, 2, (1024, 1024), 100)
    _, matched = _check([item_of(im, np.float32) for im in ims], _gt_of(ims, 106, max_shift=12))
    assert matched > 10


def test_ap_4k_image(cuda_device):
    ims = synth.make_batch(107, 1, (2160, 3840), 50, max_instances=50)
    _check([item_of(im, np.float32) for im in ims], _gt_of(ims, 108), with_ap=False)


def test_mixed_shapes_no_predictions_and_no_gt(cuda_device):
    rng = np.random.default_rng(109)
    ims = [synth.make_image(rng, hw, n, num_classes=5, max_instances=24)
           for hw, n in [((120, 200), 20), ((64, 64), 0), ((333, 75), 24), ((90, 90), 7)]]
    gts = _gt_of(ims, 110)
    gts[3] = (np.zeros((0, 4), np.int32), np.zeros(0, np.int32), np.zeros((90, 90, 0), bool))
    got, _ = _check([item_of(im, np.float32) for im in ims], gts, np.arange(0.5, 1.0, 0.05))
    assert got[1]["overlaps"].shape == (0, gts[1][2].shape[2]) and got[1]["overlaps"].dtype == np.float64
    assert got[3]["overlaps"].dtype == np.float64 and np.isnan(got[3]["ap"]).all()


def test_duplicate_and_empty_ground_truth(cuda_device):
    """Duplicate gts (IoU ties: the larger index wins), an empty prediction matching an empty gt
    of its class (NaN IoU), trimmed zero boxes, and sets where every mask is empty."""
    rng = np.random.default_rng(111)
    ims = [synth.make_image(rng, (96, 128), 10, num_classes=4, max_instances=16) for _ in range(2)]
    ims[0].mrcnn_mask[0] = 0.0                              # kept instance 0: an empty mask
    items = [item_of(im, np.float32) for im in ims]
    ref = api_utils.unmold_detections_batch(items)
    (b0, c0, _, m0), (b1, c1, _, m1) = ref
    assert not m0[..., 0].any()
    empty = np.zeros(m0.shape[:2] + (1,), bool)
    gts = [(np.concatenate([b0, [[0, 0, 0, 0]], [[1, 1, 2, 2]]]), np.concatenate([c0, [1, c0[0]]]),
            np.concatenate([m0, empty, empty], axis=2)),
           (np.concatenate([b1, b1]), np.concatenate([c1, c1]), np.concatenate([m1, m1], axis=2))]
    got, _ = _check(items, gts, (0.5, 0.9))
    assert got[1]["gt_match"][0][:len(c1)].max() == -1      # the duplicates' copies win the ties
    # every mask empty on both sides: all NaN, matched by class
    zero = [synth.make_image(rng, (40, 56), 6, num_classes=3, max_instances=8) for _ in range(2)]
    for im in zero:
        im.mrcnn_mask[:] = 0.0
    items = [item_of(im, np.float32) for im in zero]
    gts = [(b, c, np.zeros_like(m)) for b, c, _, m in api_utils.unmold_detections_batch(items)]
    got, matched = _check(items, gts)
    assert np.isnan(got[0]["overlaps"]).all() and matched > 0


def test_routes_give_identical_overlaps_and_areas(cuda_device):
    """mrx_mask_expand_packed, mrx_mask_expand + mrx_pack_masks and the wide-tile route give the
    same overlaps; prediction areas from box regions equal masks.sum((0, 1)); a second batch on
    the same engine is scored correctly."""
    rng = np.random.default_rng(112)
    ims = [synth.make_image(rng, (300, 411), 50, num_classes=6, max_instances=64) for _ in range(3)]
    gts = _gt_of(ims, 113)
    ref = api_utils.unmold_detections_batch([item_of(im, np.float32) for im in ims])
    eng = prepared_engine(ims, 64, 6, np.float32)
    gt = eng.ground_truth([c for _, c, _ in gts], [m for _, _, m in gts])
    eng.enqueue_expand_packed()
    direct = eng.enqueue_overlaps(gt).cpu().numpy()
    areas = eng._eval_bufs["areas"][:3 * 64].view(3, 64).cpu().numpy()
    eng.enqueue_expand()
    eng.pack_masks()
    via_canvas = eng.enqueue_overlaps(gt).cpu().numpy()
    for b, (rb, _, _, rm) in enumerate(ref):
        n, m = rb.shape[0], gts[b][2].shape[2]
        assert np.array_equal(areas[b, :n], rm.sum((0, 1)))
        _same_f32(direct[b, :n, :m], via_canvas[b, :n, :m])
        _same_f32(direct[b, :n, :m], eo.compute_overlaps_masks(rm, gts[b][2]))
    # wide tiles take the canvas route inside unmold_compute_ap_batch
    wide = [synth.make_image(rng, (140, 171), 20, num_classes=4, max_instances=24, mask_hw=(24, 32))
            for _ in range(2)]
    _check([item_of(im, np.float32) for im in wide], _gt_of(wide, 114))
    # a second batch on the first engine, more and larger instances
    more = [synth.make_image(rng, (300, 411), 64, num_classes=6, max_instances=64, min_box=40,
                             max_box_frac=1.0) for _ in range(3)]
    _check([item_of(im, np.float32) for im in more], _gt_of(more, 115))
    _check([item_of(im, np.float32) for im in ims], gts)


def test_evaluate_drop_ins(cuda_device):
    rng = np.random.default_rng(116)
    ims = [synth.make_image(rng, (200, 260), 30, num_classes=4, max_instances=32)]
    (rb, rc, rs, rm), = api_utils.unmold_detections_batch([item_of(im, np.float32) for im in ims])
    gb, gc, gm = _gt_of(ims, 117)[0]
    # float masks are thresholded > .5
    soft = gm * rng.uniform(0.5, 1.0, gm.shape).astype(np.float32)
    _same_f32(evaluate.compute_overlaps_masks(rm, soft), eo.compute_overlaps_masks(rm, soft))
    for a, b in [(rm[..., :0], gm), (rm, gm[..., :0])]:
        z = evaluate.compute_overlaps_masks(a, b)
        assert z.dtype == np.float64 and z.shape == (a.shape[2], b.shape[2]) and not z.any()
    args = (gb, gc, gm, rb, rc, rs, rm)
    for thr, st in [(0.5, 0.0), (np.float64(0.7), 0.0), (0.6, 0.3)]:
        got = evaluate.compute_matches(*args, iou_threshold=thr, score_threshold=st)
        want = eo.compute_matches(*args, iou_threshold=thr, score_threshold=st)
        assert all(a.dtype == np.float64 for a in got[:2])
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        _same_f32(got[2], want[2])
    got, want = evaluate.compute_ap(*args), eo.compute_ap(*args)
    for a, b in zip(got[:3], want[:3]):
        assert np.array_equal(a, b, equal_nan=True)
    out_got, out_want = io.StringIO(), io.StringIO()
    with redirect_stdout(out_got):
        ap = evaluate.compute_ap_range(*args)
    with redirect_stdout(out_want):
        ap_want = eo.compute_ap_range(*args)
    assert ap == ap_want and out_got.getvalue() == out_want.getvalue()
    # trimmed boxes and no gt at all
    for g in [(np.zeros((3, 4)), gc[:3], gm[..., :3]), (gb[:0], gc[:0], gm[..., :0])]:
        got, want = evaluate.compute_matches(*g, rb, rc, rs, rm), eo.compute_matches(*g, rb, rc, rs, rm)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert got[2].dtype == want[2].dtype == np.float64 and got[2].shape == want[2].shape
        assert np.array_equal(evaluate.compute_ap(*g, rb, rc, rs, rm)[0],
                              eo.compute_ap(*g, rb, rc, rs, rm)[0], equal_nan=True)


def test_overlaps_above_2_to_the_24_pixels(cuda_device):
    """Past 2^24 pixels the device rounds exact counts once each: f32(i) / ((f32(a1) + f32(a2)) -
    f32(i))."""
    H, W = 4096, 4097
    a = np.zeros((H, W, 2), bool)
    a[:, :, 0] = True
    a[0, 0, 0] = False                                     # 2^24 + 4095: odd, not a float32
    a[7:4001, 3:4003, 1] = True
    b = np.zeros((H, W, 1), bool)
    b[1:, 1:4097, 0] = True
    got = evaluate.compute_overlaps_masks(a, b)
    for i in range(2):
        inter = int((a[..., i] & b[..., 0]).sum())
        a1, a2 = int(a[..., i].sum()), int(b[..., 0].sum())
        f = np.float32
        want = f(inter) / ((f(a1) + f(a2)) - f(inter))
        assert got[i, 0] == want, (i, got[i, 0], want)
