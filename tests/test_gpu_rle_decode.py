"""COCO RLE ground truth decoded on the device (mrx_rle_parse, mrx_rle_decode, then
mrx_mask_extents): the planes must equal np.packbits of the oracle's masks byte for byte, the
areas and extents the oracle's, and unmold_compute_ap_batch with RLE ground truth must return
what it returns for the same masks as bool arrays."""
import numpy as np
import pytest

import coco_oracle as co
import eval_oracle as eo
import oracle
from bbox_oracle import extract_bboxes
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, synth
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import BatchLayout, MaskBatch

from helpers import item_of, prepared_engine

pytestmark = pytest.mark.gpu


def _same_f32(a, b):
    """Equal dtype and shape, NaN in the same places, every other value bit for bit."""
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb)
    assert np.array_equal(a[~na], b[~nb]) and np.array_equal(np.signbit(a[~na]), np.signbit(b[~nb]))


def _gt_of(ims, seed, **kw):
    """Ground truth (boxes, class_ids, masks) per image: the unmolded jittered image."""
    rng = np.random.default_rng(seed)
    jit = [synth.jitter_ground_truth(im, rng, **kw) for im in ims]
    return [(b, c, m) for b, c, _, m in api_utils.unmold_detections_batch(
        [item_of(im, np.float32) for im in jit])]


def _geom(H, W):
    return [H, W, H, W, 0, 0, H, W]


def _rles(masks, kind):
    """RLE dicts of bool masks [H, W, M]: 'list' (uncompressed), 'bytes' or 'str'."""
    out = []
    for k in range(masks.shape[2]):
        r = oracle.rle_encode(masks[:, :, k])
        if kind != "list":
            r["counts"] = co.rle_to_string(r["counts"])
            if kind == "str":
                r["counts"] = r["counts"].decode("ascii")
        out.append(r)
    return out


def _decode(geoms, rles, class_ids=None):
    """MaskBatch.from_rle on the current device; (batch, [planes uint8 [M_b, H_b, wb] per image],
    areas [n, R], extents [n, R, 4])."""
    import torch

    dev = torch.device("cuda", torch.cuda.current_device())
    if class_ids is None:
        class_ids = [np.ones(len(r), np.int32) for r in rles]
    gt = MaskBatch.from_rle(N.load(), dev, geoms, class_ids, rles)
    layout = BatchLayout(gt.geom, gt.R, limits=False)
    packed = gt.planes.d_packed.cpu().numpy()
    planes = []
    for b in range(gt.n):
        lo, hi = layout.packed_span(b, gt.counts[b])
        planes.append(packed[lo:hi].reshape(layout.packed_shape(b, gt.counts[b])))
    return gt, planes, gt.planes.d_areas.cpu().numpy(), gt.planes.d_extents.cpu().numpy()


def _check_masks(mask_list, kinds=("list", "bytes", "str")):
    """Decode every image's masks from each kind of RLE and compare with the oracle."""
    geoms = [_geom(*m.shape[:2]) for m in mask_list]
    for kind in kinds:
        gt, planes, areas, ext = _decode(geoms, [_rles(m, kind) for m in mask_list])
        for b, m in enumerate(mask_list):
            M = m.shape[2]
            assert np.array_equal(planes[b], np.packbits(m.transpose(2, 0, 1), axis=-1)), (kind, b)
            assert np.array_equal(areas[b, :M], m.sum((0, 1))), (kind, b)
            assert np.array_equal(ext[b, :M], extract_bboxes(m)), (kind, b)
            assert np.array_equal(gt.extents[b, :M], extract_bboxes(m)), (kind, b)


@pytest.mark.parametrize("hw,n,R,kw", [
    ((96, 128), 12, 16, {}),
    ((75, 333), 37, 40, {}),
    ((17, 9), 3, 4, dict(min_box=1, max_box_frac=1.0)),
    ((33, 1000), 7, 8, {}),
    ((1024, 1024), 100, 100, {}),
    ((800, 1333), 60, 100, {}),
    ((2160, 3840), 30, 50, {}),
])
def test_unmolded_masks(cuda_device, hw, n, R, kw):
    rng = np.random.default_rng(301)
    ims = [synth.make_image(rng, hw, n, num_classes=4, max_instances=R, **kw) for _ in range(2)]
    masks = [m for _, _, _, m in api_utils.unmold_detections_batch(
        [item_of(im, np.float32) for im in ims])]
    _check_masks(masks, ("list", "bytes") if hw[0] * hw[1] > 2 ** 20 else ("list", "bytes", "str"))


def _hand_masks(H, W):
    """All zero, all one, the four corner pixels, a run over three or more columns, a
    checkerboard."""
    m = np.zeros((H, W, 8), bool)
    m[..., 1] = True
    m[0, 0, 2] = m[0, W - 1, 3] = m[H - 1, 0, 4] = m[H - 1, W - 1, 5] = True
    f = np.zeros(H * W, bool)                     # column-major: H - 1 .. 3H + 1 spans 4 columns
    f[H - 1:min(3 * H + 2, H * W)] = True
    m[..., 6] = f.reshape((H, W), order="F")
    m[..., 7] = (np.add.outer(np.arange(H), np.arange(W)) % 2).astype(bool)
    return m


@pytest.mark.parametrize("hw", [(1, 1), (1, 37), (45, 1), (7, 5), (32, 32), (33, 65), (64, 257),
                                (129, 300)])
def test_hand_built_masks(cuda_device, hw):
    _check_masks([_hand_masks(*hw)])


def test_images_without_instances_and_kinds_mixed(cuda_device):
    """Images with M_b = 0 between others; one batch mixing bytes, str and lists gives the same
    planes as each kind alone."""
    rng = np.random.default_rng(302)
    masks = [rng.random((40, 50, 5)) < 0.3, np.zeros((30, 20, 0), bool), _hand_masks(20, 70),
             np.zeros((8, 8, 0), bool)]
    _check_masks(masks)
    geoms = [_geom(*m.shape[:2]) for m in masks]
    kinds = ["list", "bytes", "str"]
    mixed = [[_rles(m[..., k:k + 1], kinds[(b + k) % 3])[0] for k in range(m.shape[2])]
             for b, m in enumerate(masks)]
    _, planes, _, _ = _decode(geoms, mixed)
    for b, m in enumerate(masks):
        assert np.array_equal(planes[b], np.packbits(m.transpose(2, 0, 1), axis=-1)), b


def test_strings_of_the_device_encoder(cuda_device):
    """Strings from unmold_detections_rle_batch(compressed=True) decode to exactly the packed
    masks of unmold_detections_packed_batch."""
    rng = np.random.default_rng(303)
    ims = [synth.make_image(rng, hw, 20, num_classes=4, max_instances=24)
           for hw in [(120, 200), (333, 75), (64, 64)]]
    items = [item_of(im, np.float32) for im in ims]
    strings = api_utils.unmold_detections_rle_batch(items, compressed=True)
    packed = api_utils.unmold_detections_packed_batch(items)
    geoms = [_geom(*im.original_image_shape[:2]) for im in ims]
    _, planes, _, _ = _decode(geoms, [s[3] for s in strings])
    for b in range(len(ims)):
        assert np.array_equal(planes[b], packed[b][3]), b


def test_above_2_to_the_24_pixels(cuda_device):
    H, W = 4096, 4097
    m = np.zeros((H, W, 3), bool)
    m[:, :, 0] = True
    m[0, 0, 0] = False
    m[7:4001, 3:4003, 1] = True
    m[H - 1, W - 1, 2] = True
    _check_masks([m], ("list", "bytes"))


def _runs_of_intervals(intervals, total):
    """Uncompressed runs of the set pixels [start, end) (column-major positions, sorted, disjoint)."""
    runs, at = [], 0
    for s, e in intervals:
        runs += [s - at, e - s]
        at = e
    runs.append(total - at)
    return runs


def test_run_positions_past_2_to_the_31(cuda_device):
    """A 32768 x 65540 image: its runs start past 2^31 and its first count needs 7 characters."""
    H, W = 32768, 65540
    x0, x1, y0, y1 = 65000, W, 100, 32700
    ivs = [(0, 1)] + [(x * H + y0, x * H + y1) for x in range(x0, x1)] + [(H * W - 1, H * W)]
    runs = _runs_of_intervals(ivs, H * W)
    assert sum(runs[:-2]) > 2 ** 31 and runs[2] >= 2 ** 29
    wb = (W + 7) // 8
    want = np.zeros((H, wb), np.uint8)
    row = np.zeros(W, bool)
    row[x0:x1] = True
    want[y0:y1] = np.packbits(row)
    want[0, 0] |= 0x80
    want[H - 1, (W - 1) >> 3] |= 0x80 >> ((W - 1) & 7)
    for counts in (runs, co.rle_to_string(runs)):
        gt, planes, areas, ext = _decode([_geom(H, W)], [[{"size": [H, W], "counts": counts}]])
        assert np.array_equal(planes[0][0], want)
        assert areas[0, 0] == (y1 - y0) * (x1 - x0) + 2
        assert ext[0, 0].tolist() == [0, 0, H, W]
        del gt, planes


def _as_rle_gts(gts, kind="bytes", boxes=True):
    return [(b if boxes else None, c, _rles(m, kind)) for b, c, m in gts]


def _same_results(got, want, keys_extra=()):
    for g, w in zip(got, want):
        assert set(g) == set(w) | set(keys_extra)
        for key in w:
            if key == "overlaps" and w[key].dtype == np.float32:
                _same_f32(g[key], w[key])
            else:
                assert g[key].dtype == w[key].dtype, key
                assert np.array_equal(g[key], w[key], equal_nan=True), key


@pytest.mark.parametrize("thresholds,score_threshold", [
    ((0.5,), 0.0), (np.arange(0.5, 1.0, 0.05), 0.0), ((0.3, np.float64(0.6)), 0.4)])
def test_compute_ap_rle_equals_bool(cuda_device, thresholds, score_threshold):
    """RLE ground truth (strings and lists) gives what the same masks as bool arrays give; with
    gt_boxes=None, gt_rois is extract_bboxes of the masks and the rest equals passing those
    boxes.  Image 0 has an empty ground-truth mask before its last row (upstream trims its box
    and then keeps the first M - 1 masks, so the last one is dropped)."""
    rng = np.random.default_rng(304)
    ims = [synth.make_image(rng, hw, n, num_classes=4, max_instances=24)
           for hw, n in [((120, 200), 20), ((96, 128), 12), ((64, 64), 0)]]
    items = [item_of(im, np.float32) for im in ims]
    gts = _gt_of(ims, 305, max_shift=3, class_flip_frac=0.2)
    _, c0, m0 = gts[0]
    m0 = m0.copy()
    m0[..., -2] = False
    gts[0] = (None, c0, m0)
    gts = [(extract_bboxes(m), c, m) for _, c, m in gts]
    want = api_utils.unmold_compute_ap_batch(items, gts, thresholds, score_threshold)
    for kind in ("bytes", "list"):
        got = api_utils.unmold_compute_ap_batch(items, _as_rle_gts(gts, kind), thresholds,
                                                score_threshold)
        _same_results(got, want)
    got = api_utils.unmold_compute_ap_batch(items, _as_rle_gts(gts, "str", boxes=False),
                                            thresholds, score_threshold)
    _same_results(got, want, ["gt_rois"])
    for g, (b, _, m) in zip(got, gts):
        assert g["gt_rois"].dtype == np.int32 and np.array_equal(g["gt_rois"], extract_bboxes(m))
    assert want[0]["gt_match"].shape[1] == m0.shape[2] - 1
    # and the oracle agrees with the bool path
    for b, (g, (rb, rc, rs, rm)) in enumerate(zip(want, api_utils.unmold_detections_batch(items))):
        gm, pm, ov = eo.compute_matches(*gts[b], rb, rc, rs, rm, thresholds[0], score_threshold)
        assert np.array_equal(g["gt_match"][0], gm) and np.array_equal(g["pred_match"][0], pm)


@pytest.mark.parametrize("counts,match", [
    (b"0\x7f", "a counts character outside"),
    (b"`", "the counts string ends inside a value"),
    (co.rle_to_string([5, 2, 1, -3, 11]), "a count is negative or does not fit"),
    (co.rle_to_string([2 ** 32, 16]), "a count is negative or does not fit"),
    (b"PPPPPPP0", "a count is negative or does not fit"),           # 8 groups
    (co.rle_to_string([3, 12]), r"the counts do not sum to H\*W = 2240"),
    ([3, 12], r"the counts do not sum to H\*W = 2240"),
    (b"", r"the counts do not sum to H\*W = 2240"),
])
def test_malformed_input_raises(cuda_device, counts, match):
    """Each status kind raises ValueError naming the image and the instance; the malformed
    instance sits between valid ones of the same image, so a wrong bound could only write into
    its own plane, and a valid call on the same engine afterwards is right."""
    rng = np.random.default_rng(306)
    ims = [synth.make_image(rng, (40, 56), 6, num_classes=3, max_instances=8) for _ in range(2)]
    eng = prepared_engine(ims, 8, 3, np.float32)
    good = rng.random((40, 56, 3)) < 0.5
    rles = [_rles(good, "bytes"), _rles(good, "list")]
    rles[1][1] = {"size": [40, 56], "counts": counts}
    cls = [np.ones(3, np.int32)] * 2
    with pytest.raises(ValueError, match="image 1, instance 1: " + match):
        eng.ground_truth_rle(cls, rles)
    gt = eng.ground_truth_rle(cls, [_rles(good, "bytes"), _rles(good, "str")])
    layout = BatchLayout(gt.geom, gt.R, limits=False)
    packed = gt.planes.d_packed.cpu().numpy()
    for b in range(2):
        lo, hi = layout.packed_span(b, 3)
        assert np.array_equal(packed[lo:hi].reshape(3, 40, 7),
                              np.packbits(good.transpose(2, 0, 1), axis=-1))
