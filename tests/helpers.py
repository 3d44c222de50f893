"""Shared helpers for the parity tests (oracle = checker, CUDA path = thing under test)."""
import numpy as np

import oracle

# Stated fp32 tolerance of the resized (pre-threshold) mask values: the reference
# interpolates in float64 (inputs are widened float32, serve.py:131-136); the device does
# two fp32 lerps (|err| <~ 3e-7 for values in [0,1]).
MASK_VALUE_ATOL = 1e-6


def oracle_unmold(im, dtype=np.float64, return_resized=False):
    return oracle.unmold_detections(
        im.detections.astype(dtype), im.mrcnn_mask.astype(dtype),
        im.original_image_shape, im.image_shape, im.window, return_resized=return_resized)


def item_of(im, dtype=np.float64):
    return (im.detections.astype(dtype), im.mrcnn_mask.astype(dtype),
            im.original_image_shape, im.image_shape, im.window)


def compare_masks(gpu_masks, ref_masks, resized, boxes):
    """Binary masks must agree everywhere the oracle's pre-threshold value is further than
    MASK_VALUE_ATOL from 0.5.  Returns (n_flips_outside_band, n_pixels_in_band)."""
    assert gpu_masks.shape == ref_masks.shape, (gpu_masks.shape, ref_masks.shape)
    assert gpu_masks.dtype == np.bool_
    diff = gpu_masks != ref_masks
    in_band = 0
    bad = 0
    if diff.any():
        for i, (y1, x1, y2, x2) in enumerate(boxes):
            d = diff[y1:y2, x1:x2, i]
            if d.any():
                near = np.abs(resized[i] - 0.5) <= MASK_VALUE_ATOL
                bad += int((d & ~near).sum())
        # differences outside any box are always errors
        outside = diff.copy()
        for i, (y1, x1, y2, x2) in enumerate(boxes):
            outside[y1:y2, x1:x2, i] = False
        bad += int(outside.sum())
    for r in resized:
        in_band += int((np.abs(r - 0.5) <= MASK_VALUE_ATOL).sum())
    return bad, in_band


def mask_parity_stats(gpu_masks, ref_masks, resized, boxes):
    """Everything the parity contract talks about, for one image: number of mask pixels that
    differ from the oracle outside / inside the +-MASK_VALUE_ATOL band around the threshold,
    number of in-box pixels inside the band, number of pixels compared."""
    assert gpu_masks.shape == ref_masks.shape, (gpu_masks.shape, ref_masks.shape)
    diff = gpu_masks != ref_masks
    flips_out = flips_in = band = 0
    outside = diff.copy()
    for i, (y1, x1, y2, x2) in enumerate(boxes):
        near = np.abs(resized[i] - 0.5) <= MASK_VALUE_ATOL
        band += int(near.sum())
        d = diff[y1:y2, x1:x2, i]
        if d.any():
            flips_out += int((d & ~near).sum())
            flips_in += int((d & near).sum())
        outside[y1:y2, x1:x2, i] = False
    flips_out += int(outside.sum())          # a set pixel outside its box is always an error
    return {"flips_outside_band": flips_out, "flips_inside_band": flips_in,
            "band_pixels": band, "pixels": int(gpu_masks.size)}


def value_parity_stats(values, resized, boxes):
    """values: float32 [H,W,N] pre-threshold samples the production kernel stored (only in-box
    elements are meaningful).  Returns max |gpu - oracle| over every in-box sample and the
    sample count."""
    worst, count = 0.0, 0
    for i, (y1, x1, y2, x2) in enumerate(boxes):
        v = values[y1:y2, x1:x2, i].astype(np.float64)
        err = np.abs(v - resized[i])
        if err.size:
            worst = max(worst, float(err.max()))
            count += err.size
    return {"max_abs_err": worst, "samples": count}


def record_stats(name, stats):
    """Append one line to the JSONL file named by MRX_PARITY_STATS (nothing when it is unset)."""
    import json
    import os

    path = os.environ.get("MRX_PARITY_STATS")
    if not path:
        return
    try:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "a") as f:
            f.write(json.dumps({"case": name, **stats}) + "\n")
    except OSError:
        pass
