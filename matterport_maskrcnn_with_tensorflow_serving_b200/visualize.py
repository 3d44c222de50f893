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
(`find_contours` of each padded mask, traced on the device, DESIGN.md section 3.11).

With `annotate=True` the boxes, contour outlines and captions are drawn too, as OpenCV draws
them at the image's own resolution (DESIGN.md section 3.25): `cv2.rectangle` and
`cv2.polylines(..., shift=1)` in each instance's colour, `cv2.putText` captions in white.  The
outlines and boxes are rasterised on the device (`mrx_annotate_draw` / `_resolve`); the captions
are shaped by cv2 on the host (`caption_patches`) and only their stencil bits go to the device.
matplotlib's figure, dashes, alpha and font are not reproduced (DESIGN.md section 7).
"""
from __future__ import annotations

import colorsys
import random as _random

import numpy as np

from . import _native as N
from .engine import (BatchLayout, _download_contours, annotate_overlays, contours_to_lists,
                     trace_packed_contours)


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


# ------------------------------------------------------------------ annotations (DESIGN §3.25)
CAPTION_FONT = 0          # cv2.FONT_HERSHEY_SIMPLEX
CAPTION_SCALE = 0.5
CAPTION_DY = 8            # upstream: ax.text(x1, y1 + 8, caption)
CAPTION_MARGIN = 4        # pixels around cv2.getTextSize's box that a caption patch also covers


def color_table(colors, R):
    """[R, 3] uint8: the colour cv2 draws for the scalar `255.0 * c` of each RGB triple (rows past
    the list are 0): cvRound (half to even), a value outside int32 becoming INT_MIN, then saturated
    to [0, 255]."""
    tab = np.zeros((R, 3), dtype=np.uint8)
    for i, col in enumerate(colors[:R]):
        for c in range(3):
            v = np.rint(255.0 * float(col[c]))
            tab[i, c] = 0 if not (-2.0 ** 31 <= v < 2.0 ** 31) else min(max(int(v), 0), 255)
    return tab


def segment_pixels(p0, p1, H, W):
    """The pixels `cv2.polylines(img, [np.int32(2 * [p0, p1])], False, col, 1, cv2.LINE_8,
    shift=1)` sets for one contour segment, a step of (±½, ±½), (±1, 0) or (0, ±1) between
    integer-or-half (x, y) points: its two end points rounded half up, those inside the image.  So
    an outline is the set of its rounded vertices; mrx_annotate_draw sets exactly those."""
    out = set()
    for x, y in (p0, p1):
        px, py = (int(round(2 * x)) + 1) >> 1, (int(round(2 * y)) + 1) >> 1
        if 0 <= px < W and 0 <= py < H:
            out.add((px, py))
    return out


def caption_strings(n, class_ids=None, class_names=None, scores=None, captions=None):
    """Upstream's caption of each of n instances: `captions[i]` when captions are given, else the
    class name followed by the score to three places when the score is non-zero."""
    if captions:
        return [captions[i] for i in range(n)]
    if n == 0:
        return []
    if class_ids is None or class_names is None:
        raise ValueError("annotate needs class_ids and class_names, or captions")
    out = []
    for i in range(n):
        label = class_names[int(class_ids[i])]
        score = scores[i] if scores is not None else None
        out.append("{} {:.3f}".format(label, score) if score else label)
    return out


def caption_patches(texts, boxes, hw):
    """Stencils of `cv2.putText(img, text, (x1, y1 + 8), FONT_HERSHEY_SIMPLEX, 0.5, (255, 255,
    255), 1, cv2.LINE_8)` for the captions of one H x W image (boxes [N, 4] (y1, x1, y2, x2); an
    all-zero box gets no caption).  Each is drawn by cv2 on a patch: its text box (getTextSize
    and baseline) with CAPTION_MARGIN pixels around it, cut to the image, so the patch meets the
    image's edge exactly where the text is clipped by it and the stencil equals the same call on
    the whole image.  Returns [(y0, x0, stencil bool [h, w])] of the patches with a set pixel."""
    import cv2

    H, W = hw
    m = CAPTION_MARGIN
    out = []
    for text, box in zip(texts, np.asarray(boxes).reshape(-1, 4)):
        if not np.any(box):
            continue
        y1, x1 = int(box[0]), int(box[1])
        x, y = x1, y1 + CAPTION_DY
        (w, h), base = cv2.getTextSize(text, CAPTION_FONT, CAPTION_SCALE, 1)
        px0, px1 = max(x - m, 0), min(x + w + m, W)
        py0, py1 = max(y - h - m, 0), min(y + base + m, H)
        if px1 <= px0 or py1 <= py0:
            continue
        patch = np.zeros((py1 - py0, px1 - px0), dtype=np.uint8)
        cv2.putText(patch, text, (x - px0, y - py0), CAPTION_FONT, CAPTION_SCALE, 255, 1,
                    cv2.LINE_8)
        if patch.any():
            out.append((py0, px0, patch > 0))
    return out


def caption_stencils(boxes, hws, class_ids=None, class_names=None, scores=None, captions=None):
    """The caption stencils of a batch, as mrx_annotate_resolve takes them.  Per image b: boxes[b]
    [N_b, 4], hws[b] = (H_b, W_b), class_ids[b] and scores[b] (or None), captions[b] (or None);
    the strings are `caption_strings`, the stencils `caption_patches`.  Returns (int64 [P, 6]
    records (image, y0, x0, h, w, byte offset), uint8 stencil bits: each patch row-major, most
    significant bit first, starting on a byte)."""
    recs, bits, off = [], [], 0
    for b, hw in enumerate(hws):
        n = int(np.asarray(boxes[b]).reshape(-1, 4).shape[0])
        texts = caption_strings(n, None if class_ids is None else class_ids[b], class_names,
                                None if scores is None else scores[b],
                                None if captions is None else captions[b])
        for y0, x0, st in caption_patches(texts, boxes[b], hw):
            packed = np.packbits(st.reshape(-1))
            recs.append((b, y0, x0, st.shape[0], st.shape[1], off))
            bits.append(packed)
            off += packed.size
    return (np.array(recs, dtype=np.int64).reshape(-1, 6),
            np.concatenate(bits) if bits else np.zeros(0, dtype=np.uint8))


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
        self.colors = [colors if shared else colors[b] for b in range(B)]
        tab = np.stack([blend_table(c, alpha, engine.R) for c in self.colors])
        self.alpha = alpha
        self.d_tab = torch.from_numpy(tab).to(dev)
        self.d_off = torch.from_numpy(offs[:B].copy()).to(dev)
        self.max_px = max(H * W for H, W in hw)

    def run(self):
        eng = self.engine
        B = eng.layout.n
        N.check(self.lib.mrx_composite_masks(
            eng.d_canvas, eng.d_canvas_off, eng.d_counts, eng.d_geom, eng.d_boxes, self.d_in,
            self.d_off, self.d_tab, 1 - self.alpha, self.d_out, B, eng.R, self.max_px,
            N.stream_ptr()), "mrx_composite_masks")
        return self.outputs()

    def outputs(self):
        offs = self.offs
        return [self.d_out[int(offs[b]):int(offs[b + 1])].view(*self.layout.hw(b), 3)
                for b in range(self.layout.n)]

    def annotate(self, class_names=None, class_ids=None, scores=None, captions=None,
                 show_bbox=True):
        """Draw the boxes, outlines and captions on the overlays `run()` wrote (`composite_batch`
        with annotate=True).  The boxes, and the class ids and scores not given, are read from
        the engine (`fetch_meta`, one synchronisation)."""
        eng = self.engine
        B = self.layout.n
        counts, boxes, ids, scs = eng.fetch_meta()
        boxes = [boxes[b, :int(counts[b])] for b in range(B)]
        class_ids = class_ids if class_ids is not None else \
            [ids[b, :int(counts[b])] for b in range(B)]
        scores = scores if scores is not None else [scs[b, :int(counts[b])] for b in range(B)]
        hws = [self.layout.hw(b) for b in range(B)]
        patches = caption_stencils(boxes, hws, class_ids, class_names, scores, captions)
        rgb8 = np.stack([color_table(c, eng.R) for c in self.colors])
        eng.annotate(self.d_out, self.d_off, rgb8, patches, show_bbox)
        return self.outputs()


def composite_batch(engine, images, colors, alpha=0.5, *, annotate=False, class_names=None,
                    class_ids=None, scores=None, captions=None, show_bbox=True):
    """Overlay the masks an `UnmoldEngine` holds on its device canvas (after `enqueue`).

    images: list of uint8 HxWx3 arrays (NumPy or CUDA tensors), one per planned image, each
    of the engine's canvas size for that image.  colors: a list of RGB triples shared by all
    images, or one such list per image.  Returns a list of uint8 HxWx3 CUDA tensors.

    annotate=True also draws each kept instance's box (unless show_bbox is False), contour
    outlines and caption as OpenCV draws them (module docstring; `CompositeStage.annotate`).
    Per image b: class_ids[b] and scores[b] (default: the engine's), captions[b] (default: upstream's
    "<class_names[id]> <score:.3f>"); class_names is needed unless captions are given.
    """
    stage = CompositeStage(engine, images, colors, alpha)
    out = stage.run()
    if annotate:
        out = stage.annotate(class_names, class_ids, scores, captions, show_bbox)
    return out


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
        H * W, N.stream_ptr()), "mrx_composite_masks")
    return d_out.cpu().numpy()


def _trace_masks(boxes, masks, bufs):
    """Caller-held masks staged (`_stage_masks`), packed and traced as `mask_contours` traces
    them: (layout, device, d_counts, d_geom, (d_vertices, d_contour_off, d_inst_contour_off),
    inst_contour_off ndarray), the trace's buffers in `bufs`."""
    import torch

    lib = N.load()
    H, W = masks.shape[:2]
    n = int(boxes.shape[0])
    layout, dev, d_canvas, d_off, d_counts, d_geom = _stage_masks(
        np.ascontiguousarray(masks).astype(np.bool_, copy=False).view(np.uint8), H, W, n)
    d_packed = torch.empty(int(layout.packed_off[-1]), dtype=torch.uint8, device=dev)
    N.check(lib.mrx_pack_masks(d_canvas, d_off, d_counts, d_geom, d_packed, d_off, 1, n, H, W,
                               N.stream_ptr()), "mrx_pack_masks")
    # the whole image, or nothing for an all-zero box (display_instances skips those)
    regions = np.zeros((n, 4), dtype=np.int32)
    regions[boxes.reshape(n, -1).any(axis=1)] = (0, 0, H, W)
    d_regions = torch.from_numpy(regions).to(dev)
    d_vert, d_coff, icoff = trace_packed_contours(lib, dev, d_packed, d_off, d_counts, d_geom,
                                                  d_regions, layout, bufs=bufs)
    return layout, dev, d_counts, d_geom, (d_vert, d_coff, bufs["inst_contour_off"][:n + 1]), icoff


def _check_masks(boxes, masks):
    n = int(boxes.shape[0])
    if masks.ndim != 3 or masks.shape[-1] != n:
        raise ValueError("masks must be [H, W, N] for N boxes")
    return n


def mask_contours(boxes, masks):
    """NumPy in, NumPy out: the contour loop of `display_instances` for one image, traced on the
    device.  boxes [N,4]; masks bool [H,W,N].  Returns, per instance, the list of float64 [V, 2]
    (x, y) polygons upstream draws: `np.fliplr(v) - 1` for v in
    `skimage.measure.find_contours(padded_mask, 0.5)`, the mask padded with one pixel of zeros on
    every side; no polygon for an instance whose box is all zeros."""
    N.require_cuda()
    boxes = np.asarray(boxes)
    n = _check_masks(boxes, masks)
    if n == 0:
        return []
    layout, _, _, _, (d_vert, d_coff, _), icoff = _trace_masks(boxes, masks, {})
    verts, coff = _download_contours(d_vert, d_coff)
    return contours_to_lists(verts, coff, icoff, [n], layout)[0]


def annotate_image(image, boxes, masks, colors, class_ids=None, class_names=None, scores=None,
                   captions=None, show_bbox=True):
    """NumPy in, NumPy out: `image` (uint8 [H, W, 3], e.g. the overlay `apply_masks` returns) with
    the boxes, contour outlines (those of `mask_contours`) and captions of `display_instances`
    drawn on it as OpenCV draws them (module docstring).  boxes [N, 4]; masks bool [H, W, N];
    colors: N RGB triples."""
    import torch

    N.require_cuda()
    boxes = np.asarray(boxes)
    n = _check_masks(boxes, masks)
    image = np.ascontiguousarray(image, dtype=np.uint8)
    if n == 0:
        return image.copy()
    H, W = image.shape[:2]
    if masks.shape[:2] != (H, W):
        raise ValueError("masks must be [H, W, N] for an H x W image")
    patches = caption_stencils([boxes], [(H, W)], [class_ids], class_names, [scores], [captions])
    layout, dev, d_counts, d_geom, trace, _ = _trace_masks(boxes, masks, {})
    d_boxes = torch.from_numpy(np.ascontiguousarray(boxes, dtype=np.int32).reshape(n, 4)).to(dev)
    d_img = torch.from_numpy(image.copy()).to(dev)
    d_off = torch.zeros(1, dtype=torch.int64, device=dev)
    annotate_overlays(N.load(), dev, d_counts, d_geom, d_boxes, trace, d_img, d_off, [(H, W)], n,
                      color_table(colors, n)[None], patches, show_bbox)
    return d_img.cpu().numpy()


def display_instances(image, boxes, masks, class_ids=None, class_names=None, scores=None,
                      title="", figsize=(16, 16), ax=None, show_mask=True, show_bbox=True,
                      colors=None, captions=None, save_path=None, annotate=False):
    """Argument-compatible with the fork's `visualize.display_instances(..., save_path=)`
    (serve.py:160-169).  Computes the masked image (the pixels matplotlib would `imshow`).
    annotate=True also draws the boxes (when show_bbox), contour outlines and captions
    (`captions`, or upstream's "<class_names[class_id]> <score:.3f>") as OpenCV draws them
    (`annotate_image`); by default they are not drawn.  Returns the uint8 image; writes it to
    `save_path` when given: a `.png`, `.jpg` or `.jpeg` path gets the bytes cv2.imwrite would
    write, encoded on the device (`api_utils.encode_png_batch`, `api_utils.encode_jpeg_batch` at
    cv2's defaults); any other extension goes through cv2.imwrite."""
    n = int(boxes.shape[0])
    if n:
        assert boxes.shape[0] == masks.shape[-1]
    colors = colors or random_colors(max(n, 1))
    out = apply_masks(image, boxes, masks, colors) if (show_mask and n) else \
        np.ascontiguousarray(image).astype(np.uint8).copy()
    if annotate and n:
        out = annotate_image(out, boxes, masks, colors, class_ids, class_names, scores, captions,
                             show_bbox)
    if save_path is not None:
        path = str(save_path).lower()
        if path.endswith((".png", ".jpg", ".jpeg")):
            # the bytes cv2.imwrite would write, encoded on the device
            from . import api_utils

            encode = api_utils.encode_png_batch if path.endswith(".png") else \
                api_utils.encode_jpeg_batch
            with open(save_path, "wb") as f:
                f.write(encode([out])[0])
        else:
            import cv2

            cv2.imwrite(save_path, out[:, :, ::-1])   # OpenCV writes BGR
    return out
