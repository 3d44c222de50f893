"""COCO output made on the device (extension): the compressed RLE strings of
`unmold_detections_rle_batch(compressed=True)` must equal, byte for byte, the restated
`pycocotools.mask.encode` of the bool mask `unmold_detections` returns for the same instance, and
`unmold_coco_results_batch` / `serve.do_inference_coco_batch` must build upstream's
`build_coco_results` dicts from them."""
import json

import numpy as np
import pytest

import oracle
from coco_oracle import build_coco_results, encode, rle_to_string
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, serve, synth

from helpers import item_of, oracle_unmold

pytestmark = pytest.mark.gpu


def _check(ims, dtype=np.float32):
    """Compressed strings against the masks of unmold_detections_batch, and the default
    (uncompressed) output against the oracle's encoding of the same masks.  Returns the strings."""
    items = [item_of(im, dtype) for im in ims]
    got = api_utils.unmold_detections_rle_batch(items, compressed=True)
    runs = api_utils.unmold_detections_rle_batch(items)
    ref = api_utils.unmold_detections_batch(items)
    strings = []
    for (b, c, s, rles), (_, _, _, raw), (rb, rc, rs, rm) in zip(got, runs, ref):
        assert np.array_equal(b, rb) and np.array_equal(c, rc) and np.array_equal(s, rs)
        assert len(rles) == len(raw) == rb.shape[0]
        for i, rle in enumerate(rles):
            want = encode(rm[:, :, i])
            assert rle["size"] == want["size"] and all(type(v) is int for v in rle["size"])
            assert type(rle["counts"]) is bytes
            assert rle["counts"] == want["counts"], (i, rb[i])
            # the default output is the uncompressed encoding, as before
            assert raw[i]["counts"].dtype == np.uint32
            assert np.array_equal(raw[i]["counts"], oracle.rle_encode(rm[:, :, i])["counts"])
            assert rle_to_string(raw[i]["counts"]) == rle["counts"]
            strings.append(rle["counts"])
    return strings


@pytest.mark.parametrize("hw,n,R,kw", [
    ((96, 128), 12, 16, {}),
    ((64, 96), 40, 40, dict(min_box=60, max_box_frac=1.0)),     # full-height / full-width boxes
    ((40, 56), 30, 32, dict(min_box=20, max_box_frac=1.0)),     # boxes touching every border
    ((150, 150), 30, 32, dict(min_box=1, max_box_frac=0.1)),    # boxes smaller than the tile
    ((75, 333), 37, 40, {}),                                    # widths that are no multiple of 32
    ((33, 1000), 7, 8, {}),
    ((17, 9), 3, 4, dict(min_box=1, max_box_frac=1.0)),
    ((64, 80), 0, 4, {}),                                       # nothing detected
])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_rle_strings_equal_oracle(cuda_device, hw, n, R, kw, dtype):
    rng = np.random.default_rng(81)
    ims = [synth.make_image(rng, hw, n, num_classes=4, max_instances=R, **kw) for _ in range(3)]
    _check(ims, dtype)


def test_rle_strings_touching_the_canvas_edges(cuda_device):
    """Hand-placed boxes on the column seams of the column-major order: full canvas, full height
    at the left / right edge, bottom rows only, top rows only, first and last column only."""
    rng = np.random.default_rng(82)
    H, W = 48, 70
    boxes = [(0, 0, H, W), (0, 0, H, 9), (0, W - 11, H, W), (H - 7, 3, H, 40), (0, 5, 6, W),
             (0, W - 1, H, W), (10, 0, H, 1), (0, 20, H, 21), (H - 1, 0, H, W)]
    im = synth.make_image(rng, (H, W), len(boxes), num_classes=3, max_instances=12,
                          mold=((H, W, 3), (0, 0, H, W)))
    for i, (y1, x1, y2, x2) in enumerate(boxes):
        im.detections[i, :4] = synth._norm_boxes_f32(np.array([[y1, x1, y2, x2]], np.float64), (H, W))[0]
    im.mrcnn_mask[0] = 1.0      # instance 0 covers the canvas: its first pixel is set
    b, _, _, _ = api_utils.unmold_detections(*item_of(im, np.float32))
    assert [tuple(r) for r in b] == boxes
    strings = _check([im]) + _check([im], np.float64)
    assert strings[0] == rle_to_string([0, H * W])


def test_rle_strings_full_size_batch(cuda_device):
    """BASELINE.json configs[1] shape with a ragged second image; the strings are smaller than
    the uncompressed runs."""
    ims = synth.make_batch(83, 1, (1024, 1024), 100) + synth.make_batch(84, 1, (1024, 1024), 37)
    strings = _check(ims)
    assert len(strings) == 137
    runs = api_utils.unmold_detections_rle_batch([item_of(im, np.float32) for im in ims])
    n_runs = sum(len(r["counts"]) for _, _, _, rles in runs for r in rles)
    assert sum(len(s) for s in strings) < 4 * n_runs


def test_rle_strings_4k_image(cuda_device):
    """2160x3840: the leading run of zeros before a box reaches millions of pixels, which takes
    5 characters."""
    ims = synth.make_batch(85, 1, (2160, 3840), 20, num_classes=4, max_instances=24)
    items = [item_of(ims[0], np.float32)]
    _check(ims)
    (_, _, _, rles), = api_utils.unmold_detections_rle_batch(items)
    assert max(int(r["counts"][0]) for r in rles) >= 1 << 19       # needs 5 characters


def test_rle_strings_batch_of_empty_and_full_images(cuda_device):
    """A batch mixing images with no kept instance and images with all R kept."""
    rng = np.random.default_rng(86)
    R = 24
    ims = [synth.make_image(rng, (120, 200), n, num_classes=5, max_instances=R)
           for n in (0, R, 0, 0, R, 7)]
    got = api_utils.unmold_detections_rle_batch([item_of(im) for im in ims], compressed=True)
    assert [len(r[3]) for r in got] == [0, R, 0, 0, R, 7]
    _check(ims, np.float64)


def test_coco_results_equal_oracle(cuda_device):
    """unmold_coco_results_batch == upstream's build_coco_results on the oracle's unmold, one
    image id per image, through a non-identity category map; the result is JSON-ready once the
    counts are decoded."""
    rng = np.random.default_rng(87)
    ims = [synth.make_image(rng, hw, n, num_classes=7, max_instances=20)
           for hw, n in (((300, 420), 13), ((200, 200), 0), ((480, 640), 20))]
    image_ids = [1001, 7, 1003]
    cats = [0, 1, 3, 5, 7, 9, 90]
    got = api_utils.unmold_coco_results_batch([item_of(im) for im in ims], image_ids, cats)
    want = []
    for image_id, im in zip(image_ids, ims):
        want += build_coco_results([image_id], *oracle_unmold(im), category_ids=cats)
    assert len(got) == len(want) == 33
    for g, w in zip(got, want):
        assert g.keys() == w.keys()
        assert g["image_id"] == w["image_id"]
        assert type(g["category_id"]) is int and g["category_id"] == w["category_id"]
        assert all(type(v) is int for v in g["bbox"]) and g["bbox"] == w["bbox"]
        assert type(g["score"]) is float and g["score"] == w["score"]
        assert g["segmentation"] == w["segmentation"]
    for g in got:
        g["segmentation"]["counts"] = g["segmentation"]["counts"].decode("ascii")
    back = json.loads(json.dumps(got))
    assert back[0]["segmentation"]["counts"] == want[0]["segmentation"]["counts"].decode("ascii")
    # identity categories by default
    got = api_utils.unmold_coco_results_batch([item_of(ims[0])], ["a"])
    assert [r["category_id"] for r in got] == [int(c) for c in oracle_unmold(ims[0])[1]]
    assert {r["image_id"] for r in got} == {"a"}
    with pytest.raises(ValueError):
        api_utils.unmold_coco_results_batch([item_of(ims[0])], [1, 2])


def test_do_inference_coco_batch_matches_single_calls(cuda_device):
    """serve.do_inference_coco_batch around an injected TF-Serving call: images of different
    sizes in one batch give, per image, what a call with that image alone gives, and what the
    oracle's unmold and build_coco_results give."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import configs as cf

    rng = np.random.default_rng(88)
    imgs = [synth.synth_rgb_image(rng, 300, 420), synth.synth_rgb_image(rng, 640, 640),
            synth.synth_rgb_image(rng, 222, 150)]
    outs = []
    for img, n in zip(imgs, (11, 0, 5)):
        molded, meta, anchors, window = serve.preprocess_input(img, cf.IMAGE_SIZE, np.float32)
        outs.append((synth.make_image(rng, img.shape[:2], n, num_classes=cf.OUT_MASK_SHAPE[-1],
                                      max_instances=cf.OUT_DETECTION_SHAPE[0],
                                      mold=(molded.shape, window)), molded.shape, window))
    calls = {"k": 0}

    def predict(molded_f32, meta_f32, anchors_f32):
        im = outs[calls["k"] % len(outs)][0]
        calls["k"] += 1
        return im.detections.reshape(-1).tolist(), im.mrcnn_mask.reshape(-1).tolist()

    ids = [31, 32, 33]
    cats = list(range(100, 100 + cf.OUT_MASK_SHAPE[-1]))
    serve.set_predict_fn(predict)
    try:
        batch = serve.do_inference_coco_batch(imgs, ids, cats)
        singles = []
        for k, (img, image_id) in enumerate(zip(imgs, ids)):
            calls["k"] = k
            singles += serve.do_inference_coco_batch([img], [image_id], cats)
        assert serve.do_inference_coco_batch([], []) == []
    finally:
        serve.set_predict_fn(None)
    assert len(batch) == 16 and batch == singles
    want = []
    for image_id, img, (im, mshape, window) in zip(ids, imgs, outs):
        rb, rc, rs, rm = oracle.unmold_detections(
            im.detections.astype(np.float64), im.mrcnn_mask.astype(np.float64), img.shape,
            mshape, window)
        want += build_coco_results([image_id], rb, rc, rs, rm, category_ids=cats)
    assert [r["segmentation"] for r in batch] == [w["segmentation"] for w in want]
    assert [r["bbox"] for r in batch] == [w["bbox"] for w in want]
    assert [r["category_id"] for r in batch] == [w["category_id"] for w in want]
    assert [r["score"] for r in batch] == [w["score"] for w in want]
