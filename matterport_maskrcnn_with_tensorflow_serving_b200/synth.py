"""Seeded synthetic detections in the shape TF-Serving returns them to serve.py.

The reference decodes `mrcnn_detection` [R,6] and `mrcnn_mask` [R,28,28,C] from the
PredictResponse (serve.py:131-136) and hands them to
`unmold_detections` together with the molded-image shape and window produced by
`preprocess_input` (serve.py:83-107, :147-154).  This module fabricates exactly those
arrays (SURVEY.md section 8d) so tests, smoke() and bench.py feed the oracle and the
CUDA path identical inputs.  It has no dependency on the oracle or on the GPU.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


def square_mold_geometry(orig_h, orig_w, min_dim=800, max_dim=1024, min_scale=0):
    """Molded shape + window the reference's `resize_image(mode='square')` yields for
    an original (h, w) image (serve.py:91-97).  Pure integer/py-float host logic."""
    h, w = int(orig_h), int(orig_w)
    scale = 1
    if min_dim:
        scale = max(1, min_dim / min(h, w))
    if min_scale and scale < min_scale:
        scale = min_scale
    if max_dim:
        image_max = max(h, w)
        if round(image_max * scale) > max_dim:
            scale = max_dim / image_max
    if scale != 1:
        h, w = round(h * scale), round(w * scale)
    top = (max_dim - h) // 2
    left = (max_dim - w) // 2
    window = (top, left, h + top, w + left)
    return (max_dim, max_dim, 3), window, scale


@dataclass
class SynthImage:
    detections: np.ndarray        # [R, 6] float32  (y1,x1,y2,x2,class_id,score) normalised
    mrcnn_mask: np.ndarray        # [R, 28, 28, C] float32
    original_image_shape: tuple   # (H, W, 3)
    image_shape: tuple            # molded (Hm, Wm, 3)
    window: tuple                 # (y1, x1, y2, x2) in molded pixels
    n_valid: int


def _norm_boxes_f32(boxes, shape):
    h, w = shape
    scale = np.array([h - 1, w - 1, h - 1, w - 1], dtype=np.float64)
    shift = np.array([0, 0, 1, 1], dtype=np.float64)
    return ((boxes - shift) / scale).astype(np.float32)


def make_image(rng, orig_hw, n_valid, num_classes=81, max_instances=100,
               zero_area_rows=(), mask_hw=28, min_box=8, max_box_frac=0.5,
               mold=None):
    """One image worth of synthetic model output.

    Boxes are drawn as integer pixel boxes inside the window of the molded image
    (as TF's DetectionLayer clips them), then mapped to normalised coordinates the
    way `norm_boxes` does, stored as float32 (the wire dtype, serve.py:131).  Rows
    past `n_valid` are all-zero padding (class_id 0 terminates, upstream semantics).
    `zero_area_rows` are indices (< n_valid) forced to x2 == x1 so that the
    zero-area filter fires.  `mask_hw` is the tile side, or an (mh, mw) pair.
    """
    H, W = int(orig_hw[0]), int(orig_hw[1])
    if mold is None:
        image_shape, window, _ = square_mold_geometry(H, W)
    else:
        image_shape, window = mold
    wy1, wx1, wy2, wx2 = window
    wh, ww = wy2 - wy1, wx2 - wx1
    R = int(max_instances)
    det = np.zeros((R, 6), dtype=np.float32)
    n = int(n_valid)
    if n > 0:
        hi_h = max(min_box, int(wh * max_box_frac))
        hi_w = max(min_box, int(ww * max_box_frac))
        bh = rng.integers(min(min_box, wh), min(hi_h, wh) + 1, size=n)
        bw = rng.integers(min(min_box, ww), min(hi_w, ww) + 1, size=n)
        y1 = wy1 + (rng.random(n) * (wh - bh + 1)).astype(np.int64)
        x1 = wx1 + (rng.random(n) * (ww - bw + 1)).astype(np.int64)
        boxes_px = np.stack([y1, x1, y1 + bh, x1 + bw], axis=1).astype(np.float64)
        for r in zero_area_rows:
            boxes_px[r, 3] = boxes_px[r, 1]
        det[:n, :4] = _norm_boxes_f32(boxes_px, image_shape[:2])
        det[:n, 4] = rng.integers(1, num_classes, size=n).astype(np.float32)
        det[:n, 5] = np.sort(rng.uniform(0.7, 1.0, size=n))[::-1].astype(np.float32)
    mh, mw = (mask_hw, mask_hw) if np.isscalar(mask_hw) else mask_hw
    masks = rng.random((R, int(mh), int(mw), num_classes), dtype=np.float32)
    return SynthImage(det, masks, (H, W, 3), tuple(image_shape), tuple(window), n)


def make_batch(seed, batch, orig_hw, n_valid, num_classes=81, max_instances=100,
               **kw):
    """`batch` images; n_valid is an int or a (lo, hi) inclusive range sampled per
    image (BASELINE.json config 3)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(batch):
        if isinstance(n_valid, (tuple, list)):
            n = int(rng.integers(n_valid[0], n_valid[1] + 1))
        else:
            n = int(n_valid)
        out.append(make_image(rng, orig_hw, n, num_classes, max_instances, **kw))
    return out


def jitter_ground_truth(im, rng, max_shift=8, class_flip_frac=0.1):
    """The same synthetic image with every valid box moved by up to `max_shift` molded-image
    pixels in y and in x (kept inside the window) and about `class_flip_frac` of the class ids
    changed: unmolded, its masks overlap the original's with IoUs spread over (0, 1], which makes
    ground truth with real matches and misses."""
    det = im.detections.copy()
    n = im.n_valid
    if n:
        shape = im.image_shape[:2]
        h, w = shape
        scale = np.array([h - 1, w - 1, h - 1, w - 1], dtype=np.float64)
        shift = np.array([0, 0, 1, 1], dtype=np.float64)
        px = np.around(det[:n, :4].astype(np.float64) * scale + shift)
        wy1, wx1, wy2, wx2 = im.window
        d = rng.integers(-max_shift, max_shift + 1, size=(n, 2))
        px[:, [0, 2]] += d[:, :1]
        px[:, [1, 3]] += d[:, 1:]
        px[:, [0, 2]] = np.clip(px[:, [0, 2]], wy1, wy2)
        px[:, [1, 3]] = np.clip(px[:, [1, 3]], wx1, wx2)
        det[:n, :4] = _norm_boxes_f32(px, shape)
        flip = rng.random(n) < class_flip_frac
        C = im.mrcnn_mask.shape[-1]
        det[:n, 4][flip] = (det[:n, 4][flip] + rng.integers(1, max(C - 1, 2), size=int(flip.sum()))
                            - 1) % max(C - 1, 1) + 1
    return SynthImage(det, im.mrcnn_mask, im.original_image_shape, im.image_shape, im.window, n)


def jitter_coco_ground_truth(im, rng, crowd_frac=0.1, **kw):
    """`jitter_ground_truth` plus the COCO annotation fields that are not the mask: about
    `crowd_frac` of the instances marked iscrowd, and annotation areas (which COCOeval's area
    ranges use instead of the mask's pixel count) drawn around and on the 32^2 and 96^2
    boundaries and across all three ranges.  Returns (SynthImage, iscrowd int [n], area
    float64 [n])."""
    jit = jitter_ground_truth(im, rng, **kw)
    n = im.n_valid
    iscrowd = (rng.random(n) < crowd_frac).astype(np.int64)
    edges = np.array([32.0 ** 2 - 1, 32.0 ** 2, 32.0 ** 2 + 0.5, 96.0 ** 2 - 0.5, 96.0 ** 2,
                      96.0 ** 2 + 1])
    spread = np.exp(rng.uniform(np.log(10.0), np.log(1e5), size=n)).round(1)
    area = np.where(rng.random(n) < 0.3, edges[rng.integers(0, edges.size, size=n)], spread)
    return jit, iscrowd, area


def synth_rgb_image(rng, h, w):
    """uint8 RGB image with smooth structure + noise (for the mold step)."""
    yy, xx = np.mgrid[0:h, 0:w]
    base = (np.sin(yy / 37.0)[..., None] * 60 + np.cos(xx / 23.0)[..., None] * 60
            + np.array([128, 110, 140])[None, None, :])
    noise = rng.integers(-40, 41, size=(h, w, 3))
    return np.clip(base + noise, 0, 255).astype(np.uint8)
