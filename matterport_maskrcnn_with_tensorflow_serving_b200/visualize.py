"""Mask overlay of `visualize.display_instances` (reference: serve.py:160-169,
`mrcnn.visualize` is un-vendored there) on the device.

The reference passes the `[H, W, N]` bool masks `unmold_detections` returned to matplotlib
code that (per instance, in order) alpha-blends a colour into the image where the mask is
set, then draws boxes, captions and contour polygons as matplotlib artists and saves a PNG.
This module does the blending part -- the only part that touches every mask byte -- with
`mrx_composite_masks`, either on masks the caller holds as NumPy arrays (`apply_masks`,
`display_instances`) or directly on the device canvas of an `UnmoldEngine`
(`composite_batch`), which avoids the 105 MB per image device -> host copy of the masks
when only the overlay is wanted.  `mask_contours` computes the contour polygons upstream draws
(`find_contours` of each padded mask, traced on the device, DESIGN.md section 3.11).  Boxes,
captions and contours are NOT drawn (matplotlib rendering is out of scope, DESIGN.md section 7).
"""
from __future__ import annotations

import colorsys
import random as _random

import numpy as np

from . import _native as N
from .engine import BatchLayout, _download_contours, contours_to_lists, trace_packed_contours


def random_colors(n, bright=True, rng=None):
    """`n` distinct colours as RGB float triples in [0, 1]: evenly spaced hues at full
    saturation, shuffled (the values upstream's `random_colors` produces).  Upstream shuffles
    with the process-global `random`; pass a `random.Random` to get a reproducible order."""
    value = 1.0 if bright else 0.7
    colors = [colorsys.hsv_to_rgb(i / n, 1, value) for i in range(n)]
    (rng or _random).shuffle(colors)
    return colors


def blend_table(colors, alpha, R):
    """[R, 3] float64 rows `alpha * color[c] * 255` in Python's (= NumPy's) evaluation order."""
    tab = np.zeros((R, 3), dtype=np.float64)
    for i, col in enumerate(colors[:R]):
        for c in range(3):
            tab[i, c] = alpha * float(col[c]) * 255
    return tab


def _is_triple(x):
    return len(x) == 3 and not hasattr(x[0], "__len__")


class CompositeStage:
    """Device-side inputs of the overlay for one planned batch (images, blend table, scratch),
    staged once; `run()` launches `mrx_composite_masks` on the engine's current canvas.  Lets a
    pipeline (or a benchmark) separate the upload of the images from the kernel."""

    def __init__(self, engine, images, colors, alpha=0.5):
        import torch

        N.require_cuda()
        self.lib = N.load()
        self.engine = engine
        self.layout = layout = engine.layout
        B = 0 if layout is None else layout.n
        if B == 0 or len(images) != B:
            raise ValueError(f"{len(images)} images for a plan of {B}")
        dev = engine.device
        hw = [layout.hw(b) for b in range(B)]
        sizes = [H * W * 3 for H, W in hw]
        offs = np.zeros(B + 1, dtype=np.int64)
        np.cumsum(sizes, out=offs[1:])
        self.offs = offs
        self.d_in = torch.empty(int(offs[-1]), dtype=torch.uint8, device=dev)
        for b, img in enumerate(images):
            t = img if torch.is_tensor(img) else torch.from_numpy(np.ascontiguousarray(img))
            if t.dtype != torch.uint8 or t.numel() != sizes[b]:
                raise ValueError(f"image {b}: expected uint8 {hw[b][0]}x{hw[b][1]}x3")
            self.d_in[int(offs[b]):int(offs[b + 1])].copy_(t.reshape(-1), non_blocking=True)
        self.d_out = torch.empty_like(self.d_in)
        shared = len(colors) > 0 and _is_triple(colors[0])
        if not shared and len(colors) != B:
            raise ValueError("colors: one list of RGB triples, or one list per image")
        tab = np.stack([blend_table(colors if shared else colors[b], alpha, engine.R)
                        for b in range(B)])
        self.alpha = alpha
        self.d_tab = torch.from_numpy(tab).to(dev)
        self.d_off = torch.from_numpy(offs[:B].copy()).to(dev)
        self.max_px = max(H * W for H, W in hw)

    def run(self, stream=None):
        eng = self.engine
        B = eng.layout.n
        N.check(self.lib.mrx_composite_masks(
            eng.d_canvas, eng.d_canvas_off, eng.d_counts, eng.d_geom, eng.d_boxes, self.d_in,
            self.d_off, self.d_tab, 1 - self.alpha, self.d_out, B, eng.R, self.max_px,
            N.stream_ptr(stream)), "mrx_composite_masks")
        offs = self.offs
        return [self.d_out[int(offs[b]):int(offs[b + 1])].view(*self.layout.hw(b), 3)
                for b in range(B)]


def composite_batch(engine, images, colors, alpha=0.5, stream=None):
    """Overlay the masks an `UnmoldEngine` holds on its device canvas (after `enqueue`).

    images: list of uint8 HxWx3 arrays (NumPy or CUDA tensors), one per planned image, each
    of the engine's canvas size for that image.  colors: a list of RGB triples shared by all
    images, or one such list per image.  Returns a list of uint8 HxWx3 CUDA tensors.
    """
    return CompositeStage(engine, images, colors, alpha).run(stream)


def _stage_masks(mask_bytes, H, W, n):
    """Caller-held masks (`mask_bytes`, the uint8 bytes of [H, W, n]) as a one-image batch on the
    current device: (layout, device, d_canvas, d_off, d_counts, d_geom); the canvas past the masks
    is zero and d_off (one zero) serves every offset argument.  The plan's limits are the expand
    kernels': the pack, contour and overlay kernels check their own and take 1-pixel sides."""
    import torch

    layout = BatchLayout([[H, W, H, W, 0, 0, H, W]], n, limits=False)
    dev = torch.device("cuda", torch.cuda.current_device())
    d_canvas = torch.zeros(int(layout.canvas_off[-1]), dtype=torch.uint8, device=dev)
    lo, hi = layout.canvas_span(0, n)
    d_canvas[lo:hi].copy_(torch.from_numpy(mask_bytes.reshape(-1)))
    d_off = torch.zeros(1, dtype=torch.int64, device=dev)
    d_counts = torch.tensor([n], dtype=torch.int32, device=dev)
    d_geom = torch.from_numpy(layout.geom).to(dev)
    return layout, dev, d_canvas, d_off, d_counts, d_geom


def apply_masks(image, boxes, masks, colors, alpha=0.5):
    """NumPy in, NumPy out: the mask loop of `display_instances` for one image.

    image uint8 [H,W,3]; boxes [N,4]; masks bool [H,W,N] (the layout `unmold_detections`
    returns, which is the device canvas layout); colors: N RGB triples.  Returns uint8 [H,W,3].
    """
    import torch

    N.require_cuda()
    lib = N.load()
    image = np.ascontiguousarray(image)
    H, W = image.shape[:2]
    n = int(boxes.shape[0])
    if masks.shape[:2] != (H, W) or masks.shape[-1] != n:
        raise ValueError("masks must be [H, W, N] for N boxes")
    if n == 0:
        return image.astype(np.uint8).copy()
    _, dev, d_canvas, d_off, d_counts, d_geom = _stage_masks(
        np.ascontiguousarray(masks).view(np.uint8), H, W, n)
    d_boxes = torch.from_numpy(np.ascontiguousarray(boxes, dtype=np.int32)).to(dev)
    d_img = torch.from_numpy(image.astype(np.uint8, copy=False)).to(dev)
    d_out = torch.empty_like(d_img)
    d_tab = torch.from_numpy(blend_table(colors, alpha, n)).to(dev)
    N.check(lib.mrx_composite_masks(
        d_canvas, d_off, d_counts, d_geom, d_boxes, d_img, d_off, d_tab, 1 - alpha, d_out, 1, n,
        H * W, N.stream_ptr(None)), "mrx_composite_masks")
    return d_out.cpu().numpy()


def mask_contours(boxes, masks):
    """NumPy in, NumPy out: the contour loop of `display_instances` for one image, traced on the
    device.  boxes [N,4]; masks bool [H,W,N].  Returns, per instance, the list of float64 [V, 2]
    (x, y) polygons upstream draws: `np.fliplr(v) - 1` for v in
    `skimage.measure.find_contours(padded_mask, 0.5)`, the mask padded with one pixel of zeros on
    every side; no polygon for an instance whose box is all zeros."""
    import torch

    N.require_cuda()
    lib = N.load()
    boxes = np.asarray(boxes)
    H, W = masks.shape[:2]
    n = int(boxes.shape[0])
    if masks.ndim != 3 or masks.shape[-1] != n:
        raise ValueError("masks must be [H, W, N] for N boxes")
    if n == 0:
        return []
    layout, dev, d_canvas, d_off, d_counts, d_geom = _stage_masks(
        np.ascontiguousarray(masks).astype(np.bool_, copy=False).view(np.uint8), H, W, n)
    d_packed = torch.empty(int(layout.packed_off[-1]), dtype=torch.uint8, device=dev)
    N.check(lib.mrx_pack_masks(d_canvas, d_off, d_counts, d_geom, d_packed, d_off, 1, n, H, W,
                               N.stream_ptr(None)), "mrx_pack_masks")
    # the whole image, or nothing for an all-zero box (display_instances skips those)
    regions = np.zeros((n, 4), dtype=np.int32)
    regions[boxes.reshape(n, -1).any(axis=1)] = (0, 0, H, W)
    d_regions = torch.from_numpy(regions).to(dev)
    d_vert, d_coff, icoff = trace_packed_contours(lib, dev, d_packed, d_off, d_counts, d_geom,
                                                  d_regions, layout)
    verts, coff = _download_contours(d_vert, d_coff)
    return contours_to_lists(verts, coff, icoff, [n], layout)[0]


def display_instances(image, boxes, masks, class_ids=None, class_names=None, scores=None,
                      title="", figsize=(16, 16), ax=None, show_mask=True, show_bbox=True,
                      colors=None, captions=None, save_path=None):
    """Argument-compatible with the fork's `visualize.display_instances(..., save_path=)`
    (serve.py:160-169).  Computes the masked image (the pixels matplotlib would `imshow`);
    boxes, captions and contours are not drawn.  Returns the uint8 image; writes it to
    `save_path` when given: a `.png` path gets the bytes cv2.imwrite would write, encoded on the
    device (`api_utils.encode_png_batch`); any other extension goes through cv2.imwrite."""
    n = int(boxes.shape[0])
    if n:
        assert boxes.shape[0] == masks.shape[-1]
    colors = colors or random_colors(max(n, 1))
    out = apply_masks(image, boxes, masks, colors) if (show_mask and n) else \
        np.ascontiguousarray(image).astype(np.uint8).copy()
    if save_path is not None:
        if str(save_path).lower().endswith(".png"):
            # the bytes cv2.imwrite would write, encoded on the device (api_utils.encode_png_batch)
            from . import api_utils

            with open(save_path, "wb") as f:
                f.write(api_utils.encode_png_batch([out])[0])
        else:
            import cv2

            cv2.imwrite(save_path, out[:, :, ::-1])   # OpenCV writes BGR
    return out
