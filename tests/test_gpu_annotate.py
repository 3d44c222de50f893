"""GPU parity of the annotated overlay (DESIGN.md section 3.25): every byte of the picture equals the
OpenCV program of tests/annotate_oracle.py run on `oracle.composite_instances` with the contours
of tests/contour_oracle.py -- through `display_instances`, the engine path and `do_inference_batch`
-- and annotate=False leaves every output as it was."""
import random

import cv2
import numpy as np
import pytest

import annotate_oracle
import contour_oracle
import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, serve, synth, visualize
from matterport_maskrcnn_with_tensorflow_serving_b200 import configs as cf
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import UnmoldEngine, make_geom

from helpers import item_of

pytestmark = pytest.mark.gpu

NAMES = ["BG", "dent", "scratch", "crack", "glass shatter", "lamp broken"]


def _expected(image, boxes, masks, colors, class_ids=None, scores=None, captions=None,
              show_bbox=True, class_names=NAMES):
    overlay = oracle.composite_instances(image, boxes, masks, colors) if boxes.shape[0] else \
        image.copy()
    return annotate_oracle.annotate(overlay, boxes, colors,
                                    contour_oracle.mask_polygons(boxes, masks), class_ids,
                                    class_names, scores, captions, show_bbox)


def _edge_masks(rng, H, W, n):
    """n masks in [H, W, n]: a full-image one (touching all four edges), blobs off each edge, and
    random ones; boxes that bound them, with x2 == W / y2 == H where they touch the far edges."""
    masks = np.zeros((H, W, n), dtype=bool)
    masks[:, :, 0] = True
    masks[: H // 3, : W // 2, 1] = True
    masks[H // 2:, W // 3:, 2] = rng.random((H - H // 2, W - W // 3)) > 0.3
    for k in range(3, n):
        y1, x1 = int(rng.integers(0, H - 2)), int(rng.integers(0, W - 2))
        y2, x2 = int(rng.integers(y1 + 1, H + 1)), int(rng.integers(x1 + 1, W + 1))
        masks[y1:y2, x1:x2, k] = rng.random((y2 - y1, x2 - x1)) > 0.4
    boxes = np.zeros((n, 4), dtype=np.int32)
    for k in range(n):
        ys, xs = np.nonzero(masks[:, :, k])
        boxes[k] = (ys.min(), xs.min(), ys.max() + 1, xs.max() + 1) if ys.size else (0, 0, 0, 0)
    return boxes, masks


@pytest.mark.parametrize("show_bbox", [True, False])
def test_display_instances_annotated(cuda_device, tmp_path, show_bbox):
    """The NumPy path: masks touching every edge, an all-zero box, overlaps, score 0."""
    rng = np.random.default_rng(61)
    H, W = 57, 83
    boxes, masks = _edge_masks(rng, H, W, 9)
    boxes[4] = 0                                   # upstream skips it: no blend, box or caption
    image = synth.synth_rgb_image(rng, H, W)
    colors = visualize.random_colors(9, rng=random.Random(2))
    class_ids = rng.integers(1, len(NAMES), size=9)
    scores = np.float32(rng.uniform(0.5, 1.0, size=9))
    scores[3] = 0.0
    want = _expected(image, boxes, masks, colors, class_ids, scores, show_bbox=show_bbox)
    path = str(tmp_path / "a.png")
    got = visualize.display_instances(image, boxes, masks, class_ids, NAMES, scores,
                                      show_bbox=show_bbox, colors=colors, save_path=path,
                                      annotate=True)
    assert np.array_equal(got, want)
    assert open(path, "rb").read() == cv2.imencode(".png", want[:, :, ::-1])[1].tobytes()
    # annotate=False: the overlay alone, as before
    plain = visualize.display_instances(image, boxes, masks, class_ids, NAMES, scores,
                                        colors=colors)
    assert np.array_equal(plain, oracle.composite_instances(image, boxes, masks, colors))


def test_display_instances_custom_captions(cuda_device):
    rng = np.random.default_rng(62)
    H, W = 40, 30
    boxes, masks = _edge_masks(rng, H, W, 5)
    image = synth.synth_rgb_image(rng, H, W)
    colors = [(1.0, 0.5 / 255, 0.2), (0.3, 1.4, -0.1), (0.0, 0.0, 1.0), (0.5, 0.5, 0.5),
              (0.1, 0.9, 0.4)]
    captions = ["", "a", "long caption off the edge", "x y", "B"]
    want = _expected(image, boxes, masks, colors, captions=captions)
    got = visualize.display_instances(image, boxes, masks, colors=colors, captions=captions,
                                      annotate=True)
    assert np.array_equal(got, want)


def _edge_image(rng, hw, R, classes):
    """A synthetic image whose first kept row covers the whole window (box (0, 0, H, W) after the
    unmold, mask all ones: it touches all four edges and lies under every other instance), with
    score 0 on the second row."""
    im = synth.make_image(rng, hw, 6, num_classes=classes, max_instances=R)
    im.detections[0, :4] = synth._norm_boxes_f32(np.array([im.window], np.float64),
                                                 im.image_shape[:2])[0]
    im.mrcnn_mask[0] = 1.0
    im.detections[1, 5] = 0.0
    return im


def test_engine_path_batch(cuda_device):
    """Mixed image sizes, an empty image, masks on every edge, boxes with x2 == W and y2 == H,
    overlapping instances, score 0, and show_bbox=False, through `composite_batch`."""
    import torch

    rng = np.random.default_rng(63)
    R, classes = 24, len(NAMES)
    ims = [_edge_image(rng, (96, 130), R, classes),
           synth.make_image(rng, (64, 48), 0, num_classes=classes, max_instances=R),
           synth.make_image(rng, (150, 110), 20, num_classes=classes, max_instances=R,
                            max_box_frac=0.9),
           _edge_image(rng, (33, 71), R, classes)]
    eng = UnmoldEngine(len(ims), R, (28, 28), classes)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims])
    d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
    images = [synth.synth_rgb_image(rng, *im.original_image_shape[:2]) for im in ims]
    colors = [visualize.random_colors(R, rng=random.Random(20 + b)) for b in range(len(ims))]
    refs = [api_utils.unmold_detections(*item_of(im, np.float32)) for im in ims]
    assert refs[1][0].shape[0] == 0
    for b in (0, 3):
        H, W = ims[b].original_image_shape[:2]
        assert tuple(refs[b][0][0]) == (0, 0, H, W)
    assert refs[3][3][:, :, 0].all()
    assert refs[0][2][1] == 0
    for show_bbox in (True, False):
        eng.enqueue(d_det, d_msk)
        outs = visualize.composite_batch(eng, images, colors, annotate=True, class_names=NAMES,
                                         show_bbox=show_bbox)
        for b, (boxes, class_ids, scores, masks) in enumerate(refs):
            want = _expected(images[b], boxes, masks, colors[b], class_ids, scores,
                             show_bbox=show_bbox)
            assert np.array_equal(outs[b].cpu().numpy(), want), (b, show_bbox)
    # the same engine, annotate=False: the overlay alone
    eng.enqueue(d_det, d_msk)
    outs = visualize.composite_batch(eng, images, colors)
    for b, (boxes, _, _, masks) in enumerate(refs):
        want = oracle.composite_instances(images[b], boxes, masks, colors[b]) \
            if boxes.shape[0] else images[b]
        assert np.array_equal(outs[b].cpu().numpy(), want)


def test_unmold_overlay_batch_annotated(cuda_device):
    rng = np.random.default_rng(64)
    ims = synth.make_batch(64, 2, (120, 160), 9, num_classes=len(NAMES), max_instances=12)
    images = [synth.synth_rgb_image(rng, 120, 160) for _ in ims]
    colors = visualize.random_colors(12, rng=random.Random(5))
    items = [item_of(im, np.float32) for im in ims]
    with pytest.raises(ValueError):
        api_utils.unmold_overlay_batch(items, images, colors, annotate=True)
    res = api_utils.unmold_overlay_batch(items, images, colors, annotate=True, class_names=NAMES)
    for (b, c, s, overlay), item, image in zip(res, items, images):
        rb, rc, rs, rm = api_utils.unmold_detections(*item)
        assert np.array_equal(overlay, _expected(image, rb, rm, colors, rc, rs))


def _fake_model(rng, imgs, n_inst):
    """Synthetic TF-Serving: per request image, detections + masks for the molded geometry
    `preprocess_input` produces, answered in call order; also the unmold item of each."""
    outs = []
    for img in imgs:
        molded, _, _, window = serve.preprocess_input(img, cf.IMAGE_SIZE, np.float32)
        im = synth.make_image(rng, img.shape[:2], n_inst, num_classes=cf.OUT_MASK_SHAPE[-1],
                              max_instances=cf.OUT_DETECTION_SHAPE[0],
                              mold=(molded.shape, window))
        outs.append((im.detections.astype(np.float64), im.mrcnn_mask.astype(np.float64),
                     img.shape, molded.shape, window))
    calls = {"k": 0}

    def predict(molded_f32, meta_f32, anchors_f32):
        item = outs[calls["k"] % len(outs)]
        calls["k"] += 1
        return item[0].reshape(-1).tolist(), item[1].reshape(-1).tolist()

    return outs, predict


@pytest.mark.parametrize("image_format", ["png", "jpeg"])
def test_do_inference_batch_annotated(cuda_device, tmp_path, image_format):
    rng = np.random.default_rng(65)
    imgs = [synth.synth_rgb_image(rng, 200, 260), synth.synth_rgb_image(rng, 150, 90)]
    items, predict = _fake_model(rng, imgs, 7)
    colors = visualize.random_colors(100, rng=random.Random(9))
    names = ["BG", *cf.DAMAGE_CLASSES]
    serve.set_predict_fn(predict)
    try:
        paths = serve.do_inference_batch(imgs, colors=colors, media_dir=str(tmp_path),
                                         image_format=image_format, annotate=True)
        plain = serve.do_inference_batch(imgs, colors=colors, media_dir=str(tmp_path),
                                         image_format=image_format)
    finally:
        serve.set_predict_fn(None)
    ext = ".png" if image_format == "png" else ".jpg"
    for path, plain_path, item, img in zip(paths, plain, items, imgs):
        rb, rc, rs, rm = api_utils.unmold_detections(*item)
        assert rb.shape[0] > 0
        want = _expected(img, rb, rm, colors, rc, rs, class_names=names)
        assert open(path, "rb").read() == cv2.imencode(ext, want[:, :, ::-1])[1].tobytes()
        base = oracle.composite_instances(img, rb, rm, colors)
        assert open(plain_path, "rb").read() == cv2.imencode(ext, base[:, :, ::-1])[1].tobytes()
