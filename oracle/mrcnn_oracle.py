"""NumPy/SciPy restatement of the reference's CPU serving path.  TEST INFRASTRUCTURE.

PARITY UNPINNED: see oracle/__init__.py.  Every function names the reference call
site it serves ([REF] = serve.py:line) and the public upstream
function whose published algorithm it restates ([UPSTREAM] = matterport/Mask_RCNN,
no line numbers because no copy is on disk to check them against).

The code is written loop-for-loop like upstream on purpose (per-instance Python
loop, one fresh canvas per instance, np.stack(axis=-1)): it doubles as the CPU
baseline that bench.py times, so it must cost what the reference's path costs.
"""
from __future__ import annotations

import math

import numpy as np
import scipy.ndimage as ndi


# --------------------------------------------------------------------------- config
class OracleConfig:
    """[UPSTREAM mrcnn/config.py] defaults; stands in for the absent
    `model_configs.mconfig` ([REF] serve.py:23, used :93-98,:102)."""

    BACKBONE = "resnet101"
    BACKBONE_STRIDES = [4, 8, 16, 32, 64]
    RPN_ANCHOR_SCALES = (32, 64, 128, 256, 512)
    RPN_ANCHOR_RATIOS = [0.5, 1, 2]
    RPN_ANCHOR_STRIDE = 1
    IMAGE_RESIZE_MODE = "square"
    IMAGE_MIN_DIM = 800
    IMAGE_MAX_DIM = 1024
    IMAGE_MIN_SCALE = 0
    MEAN_PIXEL = np.array([123.7, 116.8, 103.9])
    NUM_CLASSES = 81
    MASK_SHAPE = [28, 28]
    DETECTION_MAX_INSTANCES = 100


# --------------------------------------------------------------------------- boxes
def norm_boxes(boxes, shape):
    """[UPSTREAM utils.norm_boxes] pixel -> normalised coords, result float32.
    Reached from unmold_detections ([REF] serve.py:147) and get_anchors (:105)."""
    h, w = shape
    scale = np.array([h - 1, w - 1, h - 1, w - 1])
    shift = np.array([0, 0, 1, 1])
    return np.divide((boxes - shift), scale).astype(np.float32)


def denorm_boxes(boxes, shape):
    """[UPSTREAM utils.denorm_boxes] normalised -> pixel coords, int32.
    np.around is round-half-to-even."""
    h, w = shape
    scale = np.array([h - 1, w - 1, h - 1, w - 1])
    shift = np.array([0, 0, 1, 1])
    return np.around(np.multiply(boxes, scale) + shift).astype(np.int32)


# --------------------------------------------------------------------------- resize
def resize(image, output_shape, preserve_range=False):
    """[UPSTREAM utils.resize -> skimage.transform.resize(order=1, mode='constant',
    cval=0, clip=True, anti_aliasing=False)].  scikit-image >= 0.19 executes exactly
    this scipy call for that argument set (channel axis, if any, gets zoom 1).  The
    trailing clip to [min(in,0), max(in,0)] is a no-op for order-1 interpolation
    with a zero border and is applied anyway for fidelity.

    preserve_range=False on a float image is the identity conversion (img_as_float
    keeps float64); on uint8 the mold step always passes preserve_range=True.
    """
    image = np.asarray(image)
    if image.dtype.kind != "f":
        if not preserve_range:
            raise NotImplementedError("oracle: integer input needs preserve_range=True")
        image = image.astype(np.float64)
    output_shape = tuple(int(v) for v in output_shape)
    in_shape = image.shape
    if len(output_shape) < image.ndim:
        output_shape = output_shape + in_shape[len(output_shape):]
    if any(o == 0 for o in output_shape) or image.size == 0:
        return np.zeros(output_shape, dtype=image.dtype)
    # skimage: factors = in/out ; zoom_factors = 1/factors ; ndi.zoom(...)
    factors = np.divide(in_shape, output_shape)
    zoom_factors = [1.0 / f for f in factors]
    out = ndi.zoom(image, zoom_factors, order=1, mode="grid-constant", cval=0.0,
                   grid_mode=True)
    assert out.shape == output_shape, (out.shape, output_shape)
    lo = min(float(image.min()), 0.0)
    hi = max(float(image.max()), 0.0)
    np.clip(out, lo, hi, out=out)
    return out


def resize_explicit(image, output_shape):
    """Hand-written statement of what `resize` computes for a 2-D (or HxWxC) float
    image: bilinear, half-pixel centres  src = (dst + 0.5) * in/out - 0.5, samples
    outside [0, in-1] read 0.  Used only to cross-check `resize` (tests pin the two
    to ~1e-15), so the GPU kernel is checked against a formula, not just a library.
    """
    image = np.asarray(image, dtype=np.float64)
    ih, iw = image.shape[:2]
    oh, ow = int(output_shape[0]), int(output_shape[1])
    ys = (np.arange(oh) + 0.5) * (ih / oh) - 0.5
    xs = (np.arange(ow) + 0.5) * (iw / ow) - 0.5
    y0 = np.floor(ys).astype(np.int64)
    x0 = np.floor(xs).astype(np.int64)
    wy = (ys - y0)
    wx = (xs - x0)
    pad = np.zeros((ih + 2, iw + 2) + image.shape[2:], dtype=np.float64)
    pad[1:-1, 1:-1] = image
    y0p = y0 + 1  # index into padded image; y0 in [-1, ih-1]
    x0p = x0 + 1
    shape_w = (oh, 1) + (1,) * (image.ndim - 2)
    shape_v = (1, ow) + (1,) * (image.ndim - 2)
    wy_ = wy.reshape(shape_w)
    wx_ = wx.reshape(shape_v)
    a = pad[y0p][:, x0p]
    b = pad[y0p][:, x0p + 1]
    c = pad[y0p + 1][:, x0p]
    d = pad[y0p + 1][:, x0p + 1]
    return (1 - wy_) * ((1 - wx_) * a + wx_ * b) + wy_ * ((1 - wx_) * c + wx_ * d)


# --------------------------------------------------------------------------- unmold
def unmold_mask(mask, bbox, image_shape):
    """[UPSTREAM utils.unmold_mask] 28x28 float mask -> full-canvas bool mask."""
    threshold = 0.5
    y1, x1, y2, x2 = bbox
    mask = resize(mask, (y2 - y1, x2 - x1))
    mask = np.where(mask >= threshold, 1, 0).astype(np.bool_)
    full_mask = np.zeros(image_shape[:2], dtype=np.bool_)
    full_mask[y1:y2, x1:x2] = mask
    return full_mask


def unmold_detections(detections, mrcnn_mask, original_image_shape, image_shape,
                      window, return_resized=False):
    """[REF] serve.py:147-154 call; [UPSTREAM MaskRCNN.unmold_detections] body.

    detections: [R, 6] rows (y1, x1, y2, x2, class_id, score), normalised to the
    molded image; mrcnn_mask: [R, 28, 28, C]; window: (y1, x1, y2, x2) pixels in the
    molded image.  Returns (boxes int32 [N,4], class_ids int32 [N], scores [N],
    masks bool [H, W, N]).

    A leading unit batch dim on detections / mrcnn_mask is squeezed: serve.py:131-136
    reshapes to (-1, *cf.OUT_*_SHAPE) and `cf` is absent, so both ranks must work.

    return_resized=True additionally returns the list of pre-threshold float64
    resized masks (test hook for the stated fp32 tolerance; not upstream).
    """
    detections = np.asarray(detections)
    mrcnn_mask = np.asarray(mrcnn_mask)
    if detections.ndim == 3 and detections.shape[0] == 1:
        detections = detections[0]
    if mrcnn_mask.ndim == 5 and mrcnn_mask.shape[0] == 1:
        mrcnn_mask = mrcnn_mask[0]

    zero_ix = np.where(detections[:, 4] == 0)[0]
    N = zero_ix[0] if zero_ix.shape[0] > 0 else detections.shape[0]

    boxes = detections[:N, :4]
    class_ids = detections[:N, 4].astype(np.int32)
    scores = detections[:N, 5]
    masks = mrcnn_mask[np.arange(N), :, :, class_ids]

    window = norm_boxes(window, image_shape[:2])
    wy1, wx1, wy2, wx2 = window
    shift = np.array([wy1, wx1, wy1, wx1])
    wh = wy2 - wy1
    ww = wx2 - wx1
    scale = np.array([wh, ww, wh, ww])
    boxes = np.divide(boxes - shift, scale)
    boxes = denorm_boxes(boxes, original_image_shape[:2])

    exclude_ix = np.where(
        (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1]) <= 0)[0]
    if exclude_ix.shape[0] > 0:
        boxes = np.delete(boxes, exclude_ix, axis=0)
        class_ids = np.delete(class_ids, exclude_ix, axis=0)
        scores = np.delete(scores, exclude_ix, axis=0)
        masks = np.delete(masks, exclude_ix, axis=0)
        N = class_ids.shape[0]

    full_masks = []
    resized = []
    for i in range(N):
        if return_resized:
            y1, x1, y2, x2 = boxes[i]
            resized.append(resize(masks[i], (y2 - y1, x2 - x1)))
        full_mask = unmold_mask(masks[i], boxes[i], original_image_shape)
        full_masks.append(full_mask)
    full_masks = np.stack(full_masks, axis=-1) \
        if full_masks else np.empty(tuple(original_image_shape[:2]) + (0,))

    if return_resized:
        return boxes, class_ids, scores, full_masks, resized
    return boxes, class_ids, scores, full_masks


# --------------------------------------------------------------------------- anchors
def compute_backbone_shapes(config, image_shape):
    """[UPSTREAM model.compute_backbone_shapes] (ResNet backbones)."""
    return np.array(
        [[int(math.ceil(image_shape[0] / stride)),
          int(math.ceil(image_shape[1] / stride))]
         for stride in config.BACKBONE_STRIDES])


def generate_anchors(scales, ratios, shape, feature_stride, anchor_stride):
    """[UPSTREAM utils.generate_anchors] one pyramid level, pixel coords float64."""
    scales, ratios = np.meshgrid(np.array(scales), np.array(ratios))
    scales = scales.flatten()
    ratios = ratios.flatten()
    heights = scales / np.sqrt(ratios)
    widths = scales * np.sqrt(ratios)
    shifts_y = np.arange(0, shape[0], anchor_stride) * feature_stride
    shifts_x = np.arange(0, shape[1], anchor_stride) * feature_stride
    shifts_x, shifts_y = np.meshgrid(shifts_x, shifts_y)
    box_widths, box_centers_x = np.meshgrid(widths, shifts_x)
    box_heights, box_centers_y = np.meshgrid(heights, shifts_y)
    box_centers = np.stack(
        [box_centers_y, box_centers_x], axis=2).reshape([-1, 2])
    box_sizes = np.stack([box_heights, box_widths], axis=2).reshape([-1, 2])
    boxes = np.concatenate([box_centers - 0.5 * box_sizes,
                            box_centers + 0.5 * box_sizes], axis=1)
    return boxes


def generate_pyramid_anchors(scales, ratios, feature_shapes, feature_strides,
                             anchor_stride):
    """[UPSTREAM utils.generate_pyramid_anchors] level-major concatenation."""
    anchors = []
    for i in range(len(scales)):
        anchors.append(generate_anchors(scales[i], ratios, feature_shapes[i],
                                        feature_strides[i], anchor_stride))
    return np.concatenate(anchors, axis=0)


def get_anchors(image_shape, config=OracleConfig):
    """[REF] serve.py:105 call; [UPSTREAM MaskRCNN.get_anchors] body (memo omitted:
    it caches, it does not change values).  Returns [A, 4] float32 normalised."""
    backbone_shapes = compute_backbone_shapes(config, image_shape)
    a = generate_pyramid_anchors(
        config.RPN_ANCHOR_SCALES,
        config.RPN_ANCHOR_RATIOS,
        backbone_shapes,
        config.BACKBONE_STRIDES,
        config.RPN_ANCHOR_STRIDE)
    return norm_boxes(a, image_shape[:2])


# --------------------------------------------------------------------------- mold
def resize_image(image, min_dim=None, max_dim=None, min_scale=None, mode="square"):
    """[REF] serve.py:91-97 call; [UPSTREAM utils.resize_image] body ("crop" mode is
    random/training-only and not restated)."""
    image_dtype = image.dtype
    h, w = image.shape[:2]
    window = (0, 0, h, w)
    scale = 1
    padding = [(0, 0), (0, 0), (0, 0)]
    crop = None

    if mode == "none":
        return image, window, scale, padding, crop

    if min_dim:
        scale = max(1, min_dim / min(h, w))
    if min_scale and scale < min_scale:
        scale = min_scale

    if max_dim and mode == "square":
        image_max = max(h, w)
        if round(image_max * scale) > max_dim:
            scale = max_dim / image_max

    if scale != 1:
        image = resize(image, (round(h * scale), round(w * scale)),
                       preserve_range=True)

    if mode == "square":
        h, w = image.shape[:2]
        top_pad = (max_dim - h) // 2
        bottom_pad = max_dim - h - top_pad
        left_pad = (max_dim - w) // 2
        right_pad = max_dim - w - left_pad
        padding = [(top_pad, bottom_pad), (left_pad, right_pad), (0, 0)]
        image = np.pad(image, padding, mode='constant', constant_values=0)
        window = (top_pad, left_pad, h + top_pad, w + left_pad)
    elif mode == "pad64":
        h, w = image.shape[:2]
        assert min_dim % 64 == 0, "Minimum dimension must be a multiple of 64"
        if h % 64 > 0:
            max_h = h - (h % 64) + 64
            top_pad = (max_h - h) // 2
            bottom_pad = max_h - h - top_pad
        else:
            top_pad = bottom_pad = 0
        if w % 64 > 0:
            max_w = w - (w % 64) + 64
            left_pad = (max_w - w) // 2
            right_pad = max_w - w - left_pad
        else:
            left_pad = right_pad = 0
        padding = [(top_pad, bottom_pad), (left_pad, right_pad), (0, 0)]
        image = np.pad(image, padding, mode='constant', constant_values=0)
        window = (top_pad, left_pad, h + top_pad, w + left_pad)
    else:
        raise Exception("Mode {} not supported".format(mode))
    return image.astype(image_dtype), window, scale, padding, crop


def mold_image(images, config=OracleConfig):
    """[REF] serve.py:98; [UPSTREAM model.mold_image]: float32 cast then subtract the
    float64 MEAN_PIXEL -> float64 result (the caller casts to float32, serve.py:117)."""
    return images.astype(np.float32) - config.MEAN_PIXEL


def compose_image_meta(image_id, original_image_shape, image_shape,
                       window, scale, active_class_ids):
    """[REF] serve.py:100-103; [UPSTREAM model.compose_image_meta]."""
    meta = np.array(
        [image_id] +
        list(original_image_shape) +
        list(image_shape) +
        list(window) +
        [scale] +
        list(active_class_ids)
    )
    return meta


def preprocess_input(img, img_size=640, config=OracleConfig):
    """[REF] serve.py:83-107, statement for statement (the str-path branch :85-86 is
    file IO and omitted).  cv2 is the real library, as in the reference."""
    import cv2

    if img_size is not None:
        img = cv2.resize(img, (img_size, img_size))

    molded_image, window, scale, padding, crop = resize_image(
        img,
        min_dim=config.IMAGE_MIN_DIM,
        min_scale=config.IMAGE_MIN_SCALE,
        max_dim=config.IMAGE_MAX_DIM,
        mode=config.IMAGE_RESIZE_MODE,
    )
    molded_image = mold_image(molded_image, config)

    image_meta = compose_image_meta(
        0, img.shape, molded_image.shape, window, scale,
        np.zeros([config.NUM_CLASSES], dtype=np.int32)
    )

    anchors = get_anchors(molded_image.shape, config)

    return molded_image, image_meta, anchors, window


# =====================================================================================
# mask compositing of visualize.display_instances (serve.py:160-169)  -- SURVEY.md 8f rank 2
# =====================================================================================
def random_colors(N, bright=True, rng=None):
    """[UPSTREAM mrcnn/visualize.py random_colors] N visually distinct colours: evenly
    spaced hues in HSV converted to RGB floats in [0,1], then shuffled.  Upstream shuffles
    with the global `random` module (not reproducible); pass `rng` (a `random.Random`) to
    make the order reproducible -- the VALUES are the upstream ones."""
    import colorsys
    import random as _random

    brightness = 1.0 if bright else 0.7
    hsv = [(i / N, 1, brightness) for i in range(N)]
    colors = list(map(lambda c: colorsys.hsv_to_rgb(*c), hsv))
    (rng or _random).shuffle(colors)
    return colors


def apply_mask(image, mask, color, alpha=0.5):
    """[UPSTREAM mrcnn/visualize.py apply_mask] blend `color` into `image` where mask == 1.
    `image` is the uint32 working copy display_instances makes; NumPy evaluates the blend in
    float64 and the assignment back into the uint32 array truncates."""
    for c in range(3):
        image[:, :, c] = np.where(mask == 1,
                                  image[:, :, c] * (1 - alpha) + alpha * color[c] * 255,
                                  image[:, :, c])
    return image


def composite_instances(image, boxes, masks, colors, alpha=0.5):
    """[REF] serve.py:160-169 calls visualize.display_instances(img, boxes, masks, ...);
    [UPSTREAM] the mask part of its body: masked_image = image.astype(uint32).copy(); for
    each instance in order, skip it when its box is all zeros, else apply_mask; the figure
    shows masked_image.astype(uint8).  (Boxes, captions and contour polygons are matplotlib
    artists drawn on top: not part of this function.)  Returns the uint8 H x W x 3 image."""
    N = boxes.shape[0]
    assert masks.shape[-1] == N and len(colors) >= N
    masked_image = image.astype(np.uint32).copy()
    for i in range(N):
        if not np.any(boxes[i]):
            continue
        masked_image = apply_mask(masked_image, masks[:, :, i], colors[i], alpha)
    return masked_image.astype(np.uint8)


# =====================================================================================
# COCO run-length encoding of a mask  -- SURVEY.md 8f rank 4 (compact mask formats)
# =====================================================================================
def rle_encode(mask):
    """[PUBLISHED FORMAT, pycocotools maskApi.c rleEncode] "uncompressed RLE" of one binary
    mask [H, W]: the pixels in COLUMN-major (Fortran) order as alternating run lengths of zeros
    and ones, starting with zeros (so the list starts with 0 when the first pixel is set).
    Returns {'size': [H, W], 'counts': uint32 ndarray}.  pycocotools itself is not installed
    here; this is the definition its `frPyObjects` accepts and its `decode` inverts."""
    mask = np.asarray(mask)
    h, w = mask.shape
    flat = mask.reshape(-1, order="F").astype(np.uint8)
    change = np.flatnonzero(np.diff(np.concatenate([[0], flat]))) if flat.size else np.array([], np.int64)
    edges = np.concatenate([[0], change, [flat.size]])
    return {"size": [int(h), int(w)], "counts": np.diff(edges).astype(np.uint32)}


def rle_decode(rle):
    """Inverse of rle_encode: bool [H, W]."""
    h, w = rle["size"]
    counts = np.asarray(rle["counts"], dtype=np.int64)
    vals = np.zeros(len(counts), dtype=np.uint8)
    vals[1::2] = 1
    flat = np.repeat(vals, counts)
    assert flat.size == h * w, (flat.size, h, w)
    return flat.reshape((h, w), order="F").astype(np.bool_)
