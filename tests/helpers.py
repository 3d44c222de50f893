"""Shared helpers for the parity tests (oracle = checker, CUDA path = thing under test)."""
import dataclasses

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


def pad_rows(im, R):
    """The same image with its detections and mask tiles padded to R rows of class 0: the kept
    instances do not change, and R selects the expand kernel (team or generic)."""
    n = im.detections.shape[0]
    assert R >= n, (R, n)
    det = np.zeros((R, 6), dtype=im.detections.dtype)
    det[:n] = im.detections
    msk = np.zeros((R,) + im.mrcnn_mask.shape[1:], dtype=im.mrcnn_mask.dtype)
    msk[:n] = im.mrcnn_mask
    return dataclasses.replace(im, detections=det, mrcnn_mask=msk)


def tile_hw(mask_hw):
    """(mh, mw) of a tile side or an (mh, mw) pair."""
    return (int(mask_hw), int(mask_hw)) if np.isscalar(mask_hw) else tuple(int(v) for v in mask_hw)


def prepared_engine(ims, R, classes, dtype=np.float64, mask_hw=28, **kw):
    """An UnmoldEngine planned for `ims` (each with R detection rows) after mrx_unmold_prepare:
    boxes, counts and tiles are on the device, no mask has been expanded yet.  kw go to the
    engine (chunk_bytes, ctas_per_sm)."""
    import torch

    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import UnmoldEngine, make_geom

    eng = UnmoldEngine(len(ims), R, tile_hw(mask_hw), classes, det_dtype=dtype, mask_dtype=dtype,
                       **kw)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims])
    d_det = torch.from_numpy(np.stack([im.detections.astype(dtype) for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask.astype(dtype) for im in ims])).cuda()
    eng.enqueue(d_det, d_msk, expand=False)
    return eng


def canvas_masks(eng, b, k):
    """bool [H, W, k] host copy of image b's byte canvas."""
    return eng.canvas_view(b, k).cpu().numpy().view(np.bool_)


def run_with_values(ims, R, classes, dtype=np.float64, mask_hw=28):
    """Batch through the PRODUCTION expand kernel's instrumented instantiation
    (mrx_mask_expand_values: same template, same cull / hrow / walk code).  Returns per image
    (boxes, class_ids, masks bool [H,W,N], values float32 [H,W,N])."""
    import torch

    eng = prepared_engine(ims, R, classes, dtype, mask_hw)
    total = int(eng._offsets[len(ims)])
    d_values = torch.full((total,), float("nan"), dtype=torch.float32, device="cuda")
    eng.enqueue_expand_values(d_values)
    counts, boxes, cls, scores = eng.fetch_meta()
    out = []
    for b, im in enumerate(ims):
        k = int(counts[b])
        H, W = im.original_image_shape[:2]
        o = int(eng._offsets[b])
        v = d_values[o:o + H * W * k].view(H, W, k).cpu().numpy()
        out.append((boxes[b, :k].copy(), cls[b, :k].copy(), canvas_masks(eng, b, k), v))
    # the instrumented launch must leave the same canvas as the plain one
    eng.enqueue_expand()
    for b, im in enumerate(ims):
        assert np.array_equal(canvas_masks(eng, b, out[b][0].shape[0]), out[b][2])
    return out


def check_values(name, ims, R, classes, dtype=np.float64, mask_hw=28):
    """Pre-threshold samples of the production kernel vs the float64 oracle, every instance of
    every image: |gpu - oracle| <= 1e-6; masks equal outside the band; stats recorded."""
    got = run_with_values(ims, R, classes, dtype, mask_hw)
    tot = {"max_abs_err": 0.0, "samples": 0, "flips_outside_band": 0, "flips_inside_band": 0,
           "band_pixels": 0, "pixels": 0, "images": len(ims), "instances": 0}
    for im, (b, c, m, v) in zip(ims, got):
        rb, rc, rs, rm, rz = oracle_unmold(im, dtype, return_resized=True)
        np.testing.assert_array_equal(b, rb)
        np.testing.assert_array_equal(c, rc)
        vs = value_parity_stats(v, rz, rb)
        ms = mask_parity_stats(m, rm, rz, rb)
        tot["max_abs_err"] = max(tot["max_abs_err"], vs["max_abs_err"])
        tot["samples"] += vs["samples"]
        tot["instances"] += int(rb.shape[0])
        for k in ("flips_outside_band", "flips_inside_band", "band_pixels", "pixels"):
            tot[k] += ms[k]
        # every in-box sample was stored (the buffer was NaN-filled)
        for i, (y1, x1, y2, x2) in enumerate(rb):
            assert not np.isnan(v[y1:y2, x1:x2, i]).any()
    record_stats(name, tot)
    assert tot["max_abs_err"] <= MASK_VALUE_ATOL, tot
    assert tot["flips_outside_band"] == 0, tot
    return tot


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
