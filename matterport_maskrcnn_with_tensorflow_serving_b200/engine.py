"""Device-resident engines over the C ABI (include/mrx.h).

PyTorch tensors are used only as owners of device / pinned-host memory and for streams;
every computation on the path is a libmrx kernel launched through ctypes.

  UnmoldEngine     batched `unmold_detections` (serve.py:147-154): prologue -> class-tile
                   gather -> fused mask expand, all stream-ordered, no host sync
  MaskBatch        caller-held masks (ground truth) as packed planes, from bool arrays, COCO
                   RLE or COCO polygons, scored against an engine's masks by `mask_overlaps` / `mask_matches`
  AnchorGenerator  `get_anchors` (serve.py:105)
  Molder           the body of `preprocess_input` (serve.py:83-107): cv2.resize + resize_image
                   + mold_image
"""
from __future__ import annotations

import ctypes as C
import math
import threading
import weakref
from typing import NamedTuple

import numpy as np

from . import _native as N


def _torch():
    import torch
    return torch


def _dtype_code(np_dtype):
    dt = np.dtype(np_dtype)
    if dt == np.float32:
        return N.MRX_F32
    if dt == np.float64:
        return N.MRX_F64
    raise TypeError(f"unsupported floating dtype {dt}; use float32 or float64")


def _torch_dtype(np_dtype):
    """The torch dtype of a device tensor holding np_dtype's values (uint32 as int32 bits)."""
    torch = _torch()
    return {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64,
            np.dtype(np.int64): torch.int64, np.dtype(np.int32): torch.int32,
            np.dtype(np.uint32): torch.int32, np.dtype(np.uint8): torch.uint8}[np.dtype(np_dtype)]


def make_geom(original_image_shape, image_shape, window):
    """Pack one image's geometry the way mrx_unmold_prepare expects (8 x int32)."""
    oh, ow = int(original_image_shape[0]), int(original_image_shape[1])
    ih, iw = int(image_shape[0]), int(image_shape[1])
    wy1, wx1, wy2, wx2 = [int(v) for v in window]
    return [oh, ow, ih, iw, wy1, wx1, wy2, wx2]


def _slot_offsets(sizes, align):
    """int64 [n+1]: where each slot of `sizes` bytes rounded up to `align` starts; [n] the total."""
    off = np.zeros(len(sizes) + 1, dtype=np.int64)
    np.cumsum((sizes + align - 1) // align * align, out=off[1:])
    return off


def _part_offsets(specs):
    """int64 [k+1]: where each of k arrays, given as (shape, dtype), starts in one buffer that
    holds them one after another, each from a multiple of 16 bytes (so a kernel may read any of
    them as int4); [k] the buffer's size."""
    return _slot_offsets(np.array([int(np.prod(s)) * np.dtype(d).itemsize for s, d in specs],
                                  dtype=np.int64), 16)


def _part_views(buf, specs):
    """Typed views of the arrays of `specs` in `buf`, a uint8 NumPy array or device tensor laid
    out by `_part_offsets`."""
    host = isinstance(buf, np.ndarray)
    return [buf[a:a + int(np.prod(s)) * np.dtype(d).itemsize]
            .view(np.dtype(d) if host else _torch_dtype(d)).reshape(s)
            for (s, d), a in zip(specs, _part_offsets(specs))]


def _upload_parts(parts, device):
    """One host-to-device copy of NumPy arrays in a buffer laid out by `_part_offsets`; returns
    typed device views of the same shapes."""
    specs = [(p.shape, p.dtype) for p in parts]
    blob = np.zeros(max(int(_part_offsets(specs)[-1]), 16), np.uint8)
    for v, p in zip(_part_views(blob, specs), parts):
        v[...] = p
    return _part_views(_torch().from_numpy(blob).to(device), specs)


class BatchLayout:
    """Where the outputs of n images ([n, 8] geometry, see make_geom) with R detection rows each
    live; host only.  Byte canvas: image b owns H*W*R bytes rounded up to 256 from canvas_off[b],
    its k kept masks bool [H, W, k] first.  Packed planes: R*H*ceil(W/8) bytes rounded up to 16
    from packed_off[b], its k planes uint8 [k, H, ceil(W/8)] first.  Instance i = b*R + k indexes
    the per-instance outputs (RLE runs and strings, contours).  limits=True refuses (ValueError)
    what the expand kernels do not take: a refused batch never becomes a layout."""

    def __init__(self, geoms, R, limits=True):
        g = np.ascontiguousarray(np.asarray(geoms, dtype=np.int32).reshape(-1, N.MRX_GEOM_INTS))
        self._pixels = hw = g[:, 0].astype(np.int64) * g[:, 1]
        if limits:
            if (g[:, :4] < 2).any():
                raise ValueError("image sides must be >= 2")
            if (hw > (1 << 30)).any():
                raise ValueError("canvas larger than 2^30 pixels is not supported")
            if (hw * R >= (1 << 31) - (1 << 20)).any():
                raise ValueError("a canvas of H*W*R >= 2^31 bytes is not supported "
                                 "(32-bit chunk math)")
        self.geom, self.R, self.n = g, int(R), g.shape[0]
        self.canvas_off = _slot_offsets(hw * R, 256)
        self.packed_off = _slot_offsets(g[:, 0].astype(np.int64) * ((g[:, 1] + 7) // 8) * R, 16)
        self.max_h, self.max_w = int(g[:, 0].max(initial=0)), int(g[:, 1].max(initial=0))

    def hw(self, b):
        return int(self.geom[b, 0]), int(self.geom[b, 1])

    def canvas_span(self, b, k):
        """[start, end) of image b's [H, W, k] masks in the byte canvas."""
        H, W = self.hw(b)
        o = int(self.canvas_off[b])
        return o, o + H * W * int(k)

    def packed_shape(self, b, k):
        H, W = self.hw(b)
        return int(k), H, (W + 7) // 8

    def packed_span(self, b, k):
        """[start, end) of image b's [k, H, ceil(W/8)] planes in the packed output."""
        k, H, wb = self.packed_shape(b, k)
        o = int(self.packed_off[b])
        return o, o + k * H * wb

    def canvas_bytes(self, counts):
        """Algorithmic canvas bytes for kept counts (sum H*W*N)."""
        return int((self._pixels * np.asarray(counts, np.int64)).sum())

    def kept_instances(self, counts):
        """(b, k, i = b*R + k) of every kept instance k < counts[b], in image order."""
        for b, n_kept in enumerate(counts):
            for k in range(int(n_kept)):
                yield b, k, b * self.R + k


class UnmoldEngine:
    """Batched, device-resident `unmold_detections`.

    Work buffers for up to `max_batch` images of up to `max_instances` detection rows are
    allocated once; the canvas lives in one device buffer with a fixed-capacity slot per image
    (`layout`, a BatchLayout) so that nothing on the path depends on a host read of the kept
    counts.  It comes from mrx_device_alloc: compressible memory where the GPU grants it
    (`canvas_compressed`), so its mostly-zero lines cost fewer DRAM bytes than they hold.

    Thread safety: an engine is a set of device buffers plus the plan of the last batch; a
    plan -> enqueue -> fetch sequence must not interleave with another thread's.  Callers
    that share an engine hold `engine.lock` (an RLock) across the sequence -- `api_utils`
    does.  `release()` frees the big buffers (canvas, packed output); they are re-allocated
    on the next plan.
    """

    def __init__(self, max_batch, max_instances=100, mask_hw=(28, 28), num_classes=81,
                 det_dtype=np.float32, mask_dtype=np.float32, device=None,
                 chunk_bytes=0, ctas_per_sm=0):
        N.require_cuda()
        torch = _torch()
        self.lib = N.load()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None \
            else torch.device(device)
        self.B = int(max_batch)
        self.R = int(max_instances)
        self.mh, self.mw = int(mask_hw[0]), int(mask_hw[1])
        self.C = int(num_classes)
        self.det_dtype = np.dtype(det_dtype)
        self.mask_dtype = np.dtype(mask_dtype)
        self.chunk_bytes = int(chunk_bytes)
        self.ctas_per_sm = int(ctas_per_sm)
        if self.B < 1 or self.B > N.MRX_MAX_BATCH:
            raise ValueError(f"max_batch must be in [1, {N.MRX_MAX_BATCH}]")
        dev, i32 = self.device, torch.int32
        B, R = self.B, self.R
        self.d_boxes = torch.empty((B, R, 4), dtype=i32, device=dev)
        self.d_class_ids = torch.empty((B, R), dtype=i32, device=dev)
        self.d_scores = torch.empty((B, R), dtype=_torch_dtype(self.det_dtype), device=dev)
        self.d_src_index = torch.empty((B, R), dtype=i32, device=dev)
        self.d_counts = torch.zeros((B,), dtype=i32, device=dev)
        self.d_status = torch.zeros((B,), dtype=i32, device=dev)
        self.d_tiles = torch.empty((B, R, self.mh, self.mw), dtype=torch.float32, device=dev)
        self.d_geom = torch.zeros((B, N.MRX_GEOM_INTS), dtype=i32, device=dev)
        self.d_canvas_off = torch.zeros((B,), dtype=torch.int64, device=dev)
        # scheduler words of the expand kernels: zeroed once here, left zeroed by every launch
        self.d_sched = torch.zeros((N.MRX_SCHED_WORDS,), dtype=i32, device=dev)
        self.d_canvas = None
        self.canvas_compressed = False
        self.d_packed = None
        self.d_packed_off = None
        self._packed_off_layout = None  # the layout whose packed offsets d_packed_off holds
        self.layout = None              # BatchLayout of the planned batch
        self._contour_bufs = {}     # work and output buffers of trace_contours, grown as needed
        self._eval_bufs = {}        # prediction areas and extents of _prediction_planes
        self._overlaps = None       # (ground truth, overlaps) of the last enqueue_overlaps
        self.lock = threading.RLock()
        # pinned staging for fetch_meta (one D2H batch + one synchronisation per call)
        self._h_meta = None

    def release(self):
        """Free the canvas, the packed-output, contour and overlap buffers (the work buffers stay)."""
        with self.lock:
            self.d_canvas = None
            self.d_packed = None
            self._contour_bufs = {}
            self._eval_bufs = {}
            self._overlaps = None
            self.layout = None

    # read-only views of the planned layout (the benchmark, tools and tests read them)
    _geom_host = property(lambda self: None if self.layout is None else self.layout.geom)
    _offsets = property(lambda self: None if self.layout is None else self.layout.canvas_off)
    _n_images = property(lambda self: 0 if self.layout is None else self.layout.n)

    # ------------------------------------------------------------------ planning
    def plan(self, geoms, canvas=True):
        """Set the per-image geometry ([n,8] ints, see make_geom) and size the canvas
        (canvas=False: geometry only, for callers that want the packed output alone)."""
        torch = _torch()
        g = np.asarray(geoms, dtype=np.int32).reshape(-1, N.MRX_GEOM_INTS)
        n = g.shape[0]
        if n < 1 or n > self.B:
            raise ValueError(f"batch of {n} images does not fit max_batch={self.B}")
        layout = self.layout
        if layout is None or not np.array_equal(layout.geom, g):
            layout = BatchLayout(g, self.R)     # (raises before anything here changes)
        elif not canvas or (self.d_canvas is not None and
                            self.d_canvas.numel() >= int(layout.canvas_off[-1])):
            return      # (a plan made with canvas=False may have left a smaller canvas behind)
        total = int(layout.canvas_off[-1])
        if canvas and (self.d_canvas is None or self.d_canvas.numel() < total):
            self.d_canvas = None
            self.d_canvas, self.canvas_compressed = _device_bytes(self.lib, total, self.device)
        self.d_geom[:n].copy_(torch.from_numpy(layout.geom))
        self.d_canvas_off[:n].copy_(torch.from_numpy(layout.canvas_off[:n].copy()))
        self.layout = layout

    # ------------------------------------------------------------------ launch
    def enqueue(self, d_detections, d_mrcnn_mask, stream=None, expand=True):
        """Enqueue the three kernels for the planned batch on `stream` (no host sync).
        d_detections [n,R,6] and d_mrcnn_mask [n,R,mh,mw,C] are device tensors of the
        dtypes given at construction (d_mrcnn_mask may also be PINNED HOST memory: the class
        gather then reads the wanted elements over PCIe instead of the whole tensor being
        copied first).  expand=False stops after the class-tile gather."""
        n = self._n_images
        if n == 0:
            raise RuntimeError("call plan() first")
        torch = _torch()
        if tuple(d_detections.shape) != (n, self.R, 6) or \
                d_detections.dtype != _torch_dtype(self.det_dtype):
            raise ValueError(f"detections must be {(n, self.R, 6)} {self.det_dtype}, got "
                             f"{tuple(d_detections.shape)} {d_detections.dtype}")
        if tuple(d_mrcnn_mask.shape) != (n, self.R, self.mh, self.mw, self.C) or \
                d_mrcnn_mask.dtype != _torch_dtype(self.mask_dtype):
            raise ValueError(f"mrcnn_mask must be {(n, self.R, self.mh, self.mw, self.C)} "
                             f"{self.mask_dtype}, got {tuple(d_mrcnn_mask.shape)} "
                             f"{d_mrcnn_mask.dtype}")
        if not (d_detections.is_contiguous() and d_mrcnn_mask.is_contiguous()):
            raise ValueError("inputs must be contiguous")
        st = N.stream_ptr(stream)
        # steps 1-6 and the class-tile gather in one launch; tiles are stored by detection row
        # and found through d_src_index by the expand kernels
        N.check(self.lib.mrx_unmold_prepare(
            d_detections, _dtype_code(self.det_dtype), d_mrcnn_mask, _dtype_code(self.mask_dtype),
            n, self.R, self.mh, self.mw, self.C, self.d_geom, self.d_boxes, self.d_class_ids,
            self.d_scores, self.d_src_index, self.d_counts, self.d_status, self.d_tiles,
            self.d_sched, st),
            "mrx_unmold_prepare")
        if expand:
            self.enqueue_expand(stream)

    def enqueue_expand(self, stream=None, canvas_ptr=None, images=None):
        """Only the mask-expand kernel (boxes / tiles / counts already on the device).
        canvas_ptr: write the canvases at another base address with the planned offsets
        (an integer device address, e.g. rank 0's receive buffer mapped with mrx_peer_open).
        images=(b0, b1): only that range of the planned batch (one launch per chunk lets the
        gather of a finished chunk overlap the next one)."""
        b0, b1 = (0, self._n_images) if images is None else images
        if b1 <= b0:
            return
        base = self.d_canvas if canvas_ptr is None else int(canvas_ptr)
        N.check(self.lib.mrx_mask_expand(
            self.d_tiles[b0:], self.d_src_index[b0:], self.d_boxes[b0:], self.d_counts[b0:],
            self.d_geom[b0:], self.d_canvas_off[b0:], base, b1 - b0, self.R, self.mh, self.mw,
            self.chunk_bytes, self.ctas_per_sm, self.d_sched,
            N.stream_ptr(stream)), "mrx_mask_expand")

    def enqueue_expand_values(self, d_values, stream=None):
        """Parity instrumentation: the same kernel (second instantiation of its template) also
        stores every pre-threshold sample into d_values (float32, indexed like the canvas)."""
        n = self._n_images
        if d_values.dtype != _torch().float32 or d_values.numel() < int(self.layout.canvas_off[n]):
            raise ValueError("d_values must be float32 with one element per canvas byte")
        N.check(self.lib.mrx_mask_expand_values(
            self.d_tiles, self.d_src_index, self.d_boxes, self.d_counts, self.d_geom,
            self.d_canvas_off, self.d_canvas, d_values, n, self.R, self.mh, self.mw, self.d_sched,
            N.stream_ptr(stream)),
            "mrx_mask_expand_values")

    # ------------------------------------------------------------------ packed output
    def packed_layout(self):
        """(layout.packed_off, total bytes) of the planned batch's packed output; d_packed_off is
        uploaded once per plan, when a packed output is first wanted (not on every plan)."""
        layout = self.layout
        if layout is None:
            raise RuntimeError("plan() first")
        if self._packed_off_layout is not layout:
            self.d_packed_off = _torch().from_numpy(layout.packed_off[:-1].copy()).to(self.device)
            self._packed_off_layout = layout
        return layout.packed_off, int(layout.packed_off[-1])

    def _packed_buffer(self):
        torch = _torch()
        off, total = self.packed_layout()
        if self.d_packed is None or self.d_packed.numel() < total:
            self.d_packed = None
            self.d_packed = torch.empty((total,), dtype=torch.uint8, device=self.device)
        return off

    def enqueue_expand_packed(self, stream=None, packed_ptr=None, images=None):
        """EXTENSION (not the reference layout): the expand step writing bit-packed masks
        directly (mrx_mask_expand_packed): packed[n, y] == np.packbits(masks[y, :, n]).
        Returns (d_packed, offsets).  packed_ptr: another base address (peer memory);
        images=(b0, b1): only that range of the planned batch."""
        b0, b1 = (0, self._n_images) if images is None else images
        if packed_ptr is None:
            off = self._packed_buffer()
            base = self.d_packed
        else:
            off, _ = self.packed_layout()
            base = int(packed_ptr)
        if b1 > b0:
            N.check(self.lib.mrx_mask_expand_packed(
                self.d_tiles[b0:], self.d_src_index[b0:], self.d_boxes[b0:], self.d_counts[b0:],
                self.d_geom[b0:], self.d_packed_off[b0:], base, b1 - b0, self.R, self.mh,
                self.mw, self.layout.max_w, self.d_sched, N.stream_ptr(stream)),
                "mrx_mask_expand_packed")
        return self.d_packed, off

    def enqueue_packed(self, d_detections, d_mrcnn_mask, stream=None, direct=True):
        """prologue -> class-tile gather -> packed masks.  Returns (d_packed, offsets).
        direct=True: the expand kernel writes the bits itself (mrx_mask_expand_packed, no byte
        canvas is written) when the tiles are at most MRX_MAX_LANE_MASK_W columns wide.
        Otherwise, and for direct=False: byte canvas, then mrx_pack_masks.  Both give identical
        bytes."""
        if direct and self.mw <= N.MRX_MAX_LANE_MASK_W:
            self.enqueue(d_detections, d_mrcnn_mask, stream, expand=False)
            return self.enqueue_expand_packed(stream)
        if self.layout is not None:     # (a plan made with canvas=False has no canvas)
            self.plan(self.layout.geom, canvas=True)
        self.enqueue(d_detections, d_mrcnn_mask, stream)
        return self.pack_masks(stream)

    # ------------------------------------------------------------------ results
    def canvas_bytes(self, counts):
        return self.layout.canvas_bytes(counts)

    def canvas_view(self, b, n_kept):
        """uint8 device view [H, W, n_kept] of image b's slot (values 0/1)."""
        lo, hi = self.layout.canvas_span(b, n_kept)
        return self.d_canvas[lo:hi].view(*self.layout.hw(b), n_kept)

    def packed_view(self, b, n_kept):
        """uint8 device view [n_kept, H, ceil(W/8)] of image b's packed planes."""
        lo, hi = self.layout.packed_span(b, n_kept)
        return self.d_packed[lo:hi].view(self.layout.packed_shape(b, n_kept))

    def enqueue_rle(self, stream=None):
        """EXTENSION: COCO run-length encodings of the planned batch's masks, from the tiles
        (after `enqueue(..., expand=False)`; no mask is materialised).  Synchronises once to
        size the output.  Returns (d_run_lengths uint32 tensor, inst_off int64 ndarray [n*R+1]):
        instance i = b*R + k owns d_run_lengths[inst_off[i] + i : inst_off[i+1] + i + 1]."""
        with _stream_ctx(stream):
            d_runs, _, off = self._enqueue_rle()
        return d_runs, off

    def _enqueue_rle(self):
        """`enqueue_rle` on the current stream, also returning the device copy of inst_off:
        (d_runs, d_off, off)."""
        torch = _torch()
        n = self._n_images
        max_w = self.layout.max_w
        dev = self.device
        d_col = torch.empty((n * self.R * max_w,), dtype=torch.int32, device=dev)
        d_off = torch.empty((n * self.R + 1,), dtype=torch.int64, device=dev)
        st = N.stream_ptr(None)
        args = (self.d_tiles, self.d_src_index, self.d_boxes, self.d_counts, self.d_geom, d_col,
                d_off)
        N.check(self.lib.mrx_rle_count(*args, n, self.R, self.mh, self.mw, max_w, st),
                "mrx_rle_count")
        off = d_off.cpu().numpy()          # the one synchronisation: how many runs there are
        total = int(off[-1])
        d_pos = torch.empty((max(total, 1),), dtype=torch.int32, device=dev)
        d_runs = torch.empty((total + n * self.R,), dtype=torch.int32, device=dev)
        N.check(self.lib.mrx_rle_write(*args, d_pos, d_runs, n, self.R, self.mh,
                                       self.mw, max_w, st), "mrx_rle_write")
        return d_runs, d_off, off

    def enqueue_rle_strings(self, stream=None):
        """EXTENSION: pycocotools' compressed RLE (the "counts" string of `mask.encode`) of every
        mask of the planned batch: `enqueue_rle` (and its one synchronisation), then
        mrx_rle_strings, on `stream`.  Returns (d_str uint8, d_str_off int64 [n*R+1]) device
        tensors: instance i = b*R + k's string is d_str[d_str_off[i]:d_str_off[i+1]] (empty for
        k >= N_b), d_str_off[n*R] the total."""
        torch = _torch()
        ni = self._n_images * self.R
        with _stream_ctx(stream):
            d_runs, d_off, off = self._enqueue_rle()
            d_str = torch.empty((max(N.rle_string_bound(off[-1], ni), 1),), dtype=torch.uint8,
                                device=self.device)
            d_str_off = torch.empty((ni + 1,), dtype=torch.int64, device=self.device)
            N.check(self.lib.mrx_rle_strings(d_runs, d_off, self.d_counts,
                                             self._n_images, self.R, d_str_off, d_str,
                                             N.stream_ptr(None)), "mrx_rle_strings")
        return d_str, d_str_off

    def trace_contours(self, stream=None):
        """EXTENSION: the contour polygons of `visualize.display_instances` for every kept
        instance of the planned batch, traced on the device from the packed planes (after
        `enqueue_expand_packed` or `pack_masks`) inside each instance's box.  Synchronises to size
        the output.  Returns (d_vertices float32 [V, 2] device tensor, d_contour_off int64 device
        tensor [C + 1], inst_contour_off int64 ndarray [n*R + 1]); see `contours_to_lists`."""
        if self.layout is None or self.d_packed is None:
            raise RuntimeError("trace_contours needs the packed planes: call enqueue_expand_packed "
                               "or pack_masks first")
        return trace_packed_contours(self.lib, self.device, self.d_packed, self.d_packed_off,
                                     self.d_counts, self.d_geom, self.d_boxes, self.layout,
                                     stream, self._contour_bufs)

    def enqueue_contours(self, stream=None):
        """`trace_contours` with the result on the host: per planned image, per kept instance, the
        list of float64 [V, 2] (x, y) polygons `display_instances` draws for it."""
        d_vert, d_coff, icoff = self.trace_contours(stream)
        n = self._n_images
        with _stream_ctx(stream):
            counts = self.d_counts[:n].cpu().numpy()
            verts, coff = _download_contours(d_vert, d_coff)
        return contours_to_lists(verts, coff, icoff, counts, self.layout)

    # ------------------------------------------------------------------ scoring against ground truth
    def ground_truth(self, class_ids, masks, stream=None):
        """A `MaskBatch` of ground truth for the planned images: class_ids[b] [M_b] and bool
        masks[b] [H_b, W_b, M_b] in the plan's image shapes."""
        if self.layout is None:
            raise RuntimeError("plan() first")
        return MaskBatch(self.lib, self.device, self.layout.geom, class_ids, masks, stream)

    def ground_truth_rle(self, class_ids, rles, stream=None):
        """`ground_truth` from COCO RLE: class_ids[b] [M_b] and rles[b], a list of M_b dicts
        {'size': [H_b, W_b], 'counts': ...} (see `MaskBatch.from_rle`, which also states what
        raises), decoded on the device."""
        if self.layout is None:
            raise RuntimeError("plan() first")
        return MaskBatch.from_rle(self.lib, self.device, self.layout.geom, class_ids, rles, stream)

    def ground_truth_coco(self, class_ids, segms, stream=None):
        """`ground_truth` from COCO `segmentation` values: class_ids[b] [M_b] and segms[b], a
        list of M_b polygon lists, box lists or RLE dicts (see `MaskBatch.from_coco`, which also
        states what raises), rasterised and decoded on the device."""
        if self.layout is None:
            raise RuntimeError("plan() first")
        return MaskBatch.from_coco(self.lib, self.device, self.layout.geom, class_ids, segms,
                                   stream)

    def enqueue_overlaps(self, gt, stream=None):
        """EXTENSION: upstream `compute_overlaps_masks(pred_masks, gt_masks)` of every planned image
        against `gt` (a `MaskBatch` from `ground_truth`), on the packed planes (after
        `enqueue_expand_packed` or `pack_masks`); each prediction is read only inside its box.
        Returns the float32 device tensor [n, R, gt.R]: element (b, i, j) for i < N_b, j < M_b is
        the IoU of kept instance i and ground-truth instance j."""
        pred = self._prediction_planes(gt, "enqueue_overlaps", stream)
        self._overlaps = (gt, mask_overlaps(self.lib, pred, gt.planes, self.d_geom,
                                            self._n_images, stream))
        return self._overlaps[1]

    def enqueue_matches(self, gt, thresholds, score_threshold=0.0, stream=None):
        """EXTENSION: the matching of upstream `compute_matches` for each IoU threshold, on the
        overlaps of the last `enqueue_overlaps(gt)`.  Thresholds compare as upstream's do
        (`comparison_threshold`).  Returns device tensors (order [n, R]: rank -> kept instance,
        by score; pred_match [T, n, R] by rank: gt index or -1; gt_match [T, n, gt.R]: rank or
        -1)."""
        last = self._overlaps
        if last is None or last[0] is not gt:
            raise RuntimeError("enqueue_overlaps(gt) first")
        return mask_matches(self.lib, last[1], self.d_counts, self.d_class_ids, self.d_scores,
                            _dtype_code(self.det_dtype), gt, thresholds, score_threshold, stream)

    def predictions(self, gt=None, stream=None):
        """EXTENSION: the planned batch's kept predictions as the scorers read them
        (`coco_evaluate_batch`, `coco_boundary_evaluate_batch`, `coco_box_evaluate_batch`), after
        `enqueue`: its counts, class ids, scores and boxes.  With `gt` (a `MaskBatch` of the same
        plan, e.g. from `ground_truth_rle`) also their `Planes` on the packed planes (after
        `enqueue_expand_packed` or `pack_masks`), each prediction counted only inside its box;
        without it no mask is read, as box scoring after `enqueue(..., expand=False)` needs."""
        planes = None if gt is None else self._prediction_planes(gt, "predictions", stream)
        n = self._n_images
        if n == 0:
            raise RuntimeError("call plan() and enqueue() first")
        return Predictions(self.d_counts[:n], self.d_class_ids[:n], self.d_scores[:n],
                           self.d_boxes[:n], planes)

    def boundary_planes(self, dilation_ratio=0.02, stream=None):
        """EXTENSION: `Planes` of the boundaries of the planned batch's kept masks (after
        `enqueue_expand_packed` or `pack_masks`), as boundary_iou_api's mask_to_boundary computes
        them for `dilation_ratio`: mrx_mask_boundary inside each kept box, then mrx_mask_extents
        for the areas (the extents are the masks').  Only the bytes of a plane that hold a pixel
        of its box are written (outside the box the boundary is zero).  The buffers live in
        `_eval_bufs`."""
        if self.layout is None or self.d_packed is None:
            raise RuntimeError("boundary_planes needs the packed planes: call "
                               "enqueue_expand_packed or pack_masks first")
        d = boundary_dilation(self.layout.geom, dilation_ratio)
        with _stream_ctx(stream):
            d_dil = _torch().from_numpy(d).to(self.device)
            pred = Planes(self.d_packed, self.d_packed_off, self.d_counts, None, None, self.R)
            return mask_boundary_planes(self.lib, pred, self.d_geom, self.d_boxes, d_dil,
                                        self._n_images, self.layout.max_w, self._eval_bufs,
                                        stream)

    def _prediction_planes(self, gt, fn, stream):
        """`Planes` of the planned batch's kept instances to score against `gt` (a `MaskBatch` of
        the same plan), each counted only inside its box (mrx_mask_extents into `_eval_bufs`)."""
        if self.layout is None or self.d_packed is None:
            raise RuntimeError(f"{fn} needs the packed planes: call enqueue_expand_packed or "
                               "pack_masks first")
        n = self._n_images
        if gt.n != n or not np.array_equal(gt.geom, self.layout.geom):
            raise ValueError("the ground truth was staged for another plan")
        torch = _torch()
        bufs = self._eval_bufs
        d_areas = _buffer(bufs, "areas", n * self.R, torch.int64, self.device)
        d_ext = _buffer(bufs, "extents", n * self.R * 4, torch.int32, self.device)
        N.check(self.lib.mrx_mask_extents(
            self.d_packed, self.d_packed_off, self.d_counts, self.d_geom, self.d_boxes, d_areas,
            d_ext, n, self.R, N.stream_ptr(stream)),
            "mrx_mask_extents")
        return Planes(self.d_packed, self.d_packed_off, self.d_counts, d_areas, d_ext, self.R)

    def pack_masks(self, stream=None):
        """EXTENSION: bit-pack the byte canvases already written for the planned batch
        (mrx_pack_masks; same output layout as `enqueue_expand_packed`).  Returns
        (d_packed, offsets)."""
        n = self._n_images
        off = self._packed_buffer()
        N.check(self.lib.mrx_pack_masks(
            self.d_canvas, self.d_canvas_off, self.d_counts, self.d_geom, self.d_packed,
            self.d_packed_off, n, self.R,
            self.layout.max_h, self.layout.max_w, N.stream_ptr(stream)), "mrx_pack_masks")
        return self.d_packed, off

    def fetch_meta(self, stream=None):
        """Copy counts/status/boxes/class_ids/scores of the planned batch to the host
        (one batch of async copies into cached pinned memory, one synchronisation).
        Raises like numpy would on bad inputs.  The returned arrays are views of the
        staging buffers: valid until the next fetch_meta of this engine."""
        torch = _torch()
        n = self._n_images
        if self._h_meta is None:
            B, R = self.B, self.R
            pin = lambda shape, dt: torch.empty(shape, dtype=dt).pin_memory()  # noqa: E731
            self._h_meta = (pin((B,), torch.int32), pin((B,), torch.int32),
                            pin((B, R, 4), torch.int32), pin((B, R), torch.int32),
                            pin((B, R), _torch_dtype(self.det_dtype)))
        hc, hs, hb, hk, hsc = self._h_meta
        st = stream or torch.cuda.current_stream(self.device)
        with torch.cuda.stream(st):
            hc[:n].copy_(self.d_counts[:n], non_blocking=True)
            hs[:n].copy_(self.d_status[:n], non_blocking=True)
            hb[:n].copy_(self.d_boxes[:n], non_blocking=True)
            hk[:n].copy_(self.d_class_ids[:n], non_blocking=True)
            hsc[:n].copy_(self.d_scores[:n], non_blocking=True)
        st.synchronize()
        counts, status = hc[:n].numpy(), hs[:n].numpy()
        if (status & N.MRX_ST_CLASS_RANGE).any():
            b = int(np.nonzero(status & N.MRX_ST_CLASS_RANGE)[0][0])
            raise IndexError(f"image {b}: class id out of bounds for axis 3 with size {self.C}")
        if (status & N.MRX_ST_BOX_RANGE).any():
            b = int(np.nonzero(status & N.MRX_ST_BOX_RANGE)[0][0])
            raise ValueError(f"image {b}: a detection box falls outside the original image; "
                             "the reference's mask paste cannot broadcast it")
        return counts, hb[:n].numpy(), hk[:n].numpy(), hsc[:n].numpy()


def _device_bytes(lib, nbytes, device):
    """(uint8 tensor of `nbytes`, compressed) over memory from mrx_device_alloc on `device`.  The
    memory is freed when the last view of the tensor dies."""
    torch = _torch()
    ptr, compressed = C.c_void_p(0), C.c_int(0)
    with torch.cuda.device(device):
        N.check(lib.mrx_device_alloc(nbytes, C.byref(ptr), C.byref(compressed)),
                "mrx_device_alloc")
    owner = N.DeviceBytes(ptr.value, nbytes)
    # torch holds `owner` for as long as any view of the tensor lives; at interpreter exit the
    # driver reclaims the memory itself
    weakref.finalize(owner, _free_device_bytes, lib, ptr.value, nbytes, device).atexit = False
    return torch.as_tensor(owner, device=device), bool(compressed.value)


def _free_device_bytes(lib, ptr, nbytes, device):
    with _torch().cuda.device(device):
        N.check(lib.mrx_device_free(ptr, nbytes), "mrx_device_free")


def _buffer(bufs, name, numel, dtype, device):
    """A device tensor of at least `numel` elements kept in `bufs` (reallocated only to grow)."""
    t = bufs.get(name)
    if t is None or t.numel() < numel:
        bufs[name] = None
        t = bufs[name] = _torch().empty((max(int(numel), 1),), dtype=dtype, device=device)
    return t


class Planes(NamedTuple):
    """One side of `mask_overlaps`: packed slots (d_packed, d_packed_off), counts [n], areas
    [n, R] int64 and extents [n, R, 4] int32 of mrx_mask_extents, and the slot's R."""
    d_packed: object
    d_packed_off: object
    d_counts: object
    d_areas: object
    d_extents: object
    R: int


class Predictions(NamedTuple):
    """One batch's predictions as the COCO scorers read them: counts [n], class_ids [n, R] and
    scores [n, R] (float32 / float64), boxes [n, R, 4] (int32 (y1, x1, y2, x2) boxes, which the
    boundary scorer also takes as the regions of `planes`, or the float64 [x, y, w, h] of bbox
    results), and `Planes` of the masks for the mask scorers."""
    counts: object
    class_ids: object
    scores: object
    boxes: object
    planes: Planes = None


class MaskBatch:
    """Caller-held masks of a batch on the device as packed planes, with their areas, extents
    and class ids: class_ids[b] [M_b] and masks[b] [H_b, W_b, M_b] (bool, or thresholded `> .5`
    as upstream's compute_overlaps_masks does) for the images of `geoms` ([n, 8], see make_geom).
    Each image's bytes pass through one staging canvas sized for the largest image and are packed
    into its slot by mrx_pack_masks, so device memory holds one image's bytes plus the packed
    planes.  M_b above what mrx_pack_masks takes raises ValueError."""

    def __init__(self, lib, device, geoms, class_ids, masks, stream=None):
        torch = _torch()
        g = np.asarray(geoms, dtype=np.int32).reshape(-1, N.MRX_GEOM_INTS)
        n = g.shape[0]
        if len(masks) != n or len(class_ids) != n:
            raise ValueError(f"{len(masks)} masks and {len(class_ids)} class-id arrays for "
                             f"{n} images")
        staged, counts = [], np.zeros(n, dtype=np.int32)
        for b, (cls, m) in enumerate(zip(class_ids, masks)):
            m = np.asarray(m)
            H, W = int(g[b, 0]), int(g[b, 1])
            if m.ndim != 3 or m.shape[:2] != (H, W):
                raise ValueError(f"image {b}: masks must be [{H}, {W}, M], got {m.shape}")
            if np.shape(cls) != (m.shape[2],):
                raise ValueError(f"image {b}: {np.shape(cls)} class ids for {m.shape[2]} masks")
            m = m if m.dtype == np.bool_ else m > .5
            staged.append(np.ascontiguousarray(m).view(np.uint8))
            counts[b] = m.shape[2]

        def fill(layout, d_packed, d_off, d_zero):
            canvas = torch.empty((max(max(s.size for s in staged), 1) + 15) // 16 * 16,
                                 dtype=torch.uint8, device=device)
            for b, s in enumerate(staged):
                if s.size == 0:
                    continue
                canvas[:s.size].copy_(torch.from_numpy(s.reshape(-1)))
                H, W = layout.hw(b)
                rc = lib.mrx_pack_masks(canvas, d_zero, self.d_counts[b:],
                                        self.d_geom[b:], d_packed, d_off[b:],
                                        1, layout.R, H, W, N.stream_ptr(stream))
                if rc == N.MRX_E_UNSUPPORTED:
                    raise ValueError(lib.mrx_last_error().decode())
                N.check(rc, "mrx_pack_masks")

        self._stage(lib, device, g, class_ids, counts, [np.zeros(1, np.int64)], fill, stream)

    @classmethod
    def from_rle(cls, lib, device, geoms, class_ids, rles, stream=None):
        """The same batch from COCO RLE: rles[b] is a list of M_b dicts {'size': [H_b, W_b],
        'counts': c} with c pycocotools' compressed string (`bytes`, or an ASCII `str`) or its
        uncompressed runs (a 1-D sequence of integers in [0, 2^32), column-major, starting with
        zeros), as `annToRLE` or `mask.encode` give them; kinds may mix.  The strings and runs
        (`pack_rle`) are uploaded once and decoded on the device (mrx_rle_parse, mrx_rle_decode);
        no mask exists on the host.  Then mrx_mask_extents, and one synchronisation to read the
        status words and the extents (`extents`, int32 [n, R, 4]: what upstream's
        `extract_bboxes` returns for each mask).

        Raises ValueError naming the image and the instance for a size other than the image's, a
        counts value of another type, an uncompressed count outside [0, 2^32) and a class-id count
        other than M_b (all before anything is uploaded), and for a malformed string or runs
        found on the device: a character outside '0'..'o', a string that ends inside a value, a
        count that is negative or does not fit in uint32, or counts that do not sum to H*W.
        pycocotools decodes such input without a check; this raises instead."""
        g = np.asarray(geoms, dtype=np.int32).reshape(-1, N.MRX_GEOM_INTS)
        return cls._decoded(lib, device, g, class_ids, pack_rle(g, class_ids, rles), None, stream)

    @classmethod
    def from_coco(cls, lib, device, geoms, class_ids, segms, stream=None):
        """The same batch from COCO `segmentation` values as a COCO instances file holds them:
        segms[b] is a list of M_b of them, each a polygon list [[x0, y0, x1, y1, ...], ...], a
        box list [[x, y, w, h], ...] or an RLE dict (as for `from_rle`); kinds may mix, as crowd
        RLE sits next to polygons.  Each plane is pycocotools' `decode(annToRLE(ann))` for an
        annotation of the image's size: a polygon or box list is `frPyObjects` (polygons when the
        first part has more than 4 numbers, boxes when it has 4) merged as a union, rasterised on
        the device (mrx_poly_decode) from the scaled vertices `pack_polygons` makes; RLE dicts
        are decoded as `from_rle` decodes them.  Everything is uploaded once; one synchronisation
        reads the status words and the extents.

        Raises ValueError naming the image and the instance, before anything is uploaded, for an
        empty list, a first part of fewer than 4 numbers, a box list with a part that is not 4
        numbers, a later polygon part of fewer than 2 numbers, a coordinate that is not a finite
        number, a scaled coordinate (int)(5 * c + .5) or a difference of two consecutive ones
        outside the int range (pycocotools' behaviour is undefined for all of these but the
        first three), a value that is neither a list nor a dict, and for RLE dicts what
        `from_rle` raises.  Positions are exact for any H*W, where pycocotools' int positions
        overflow once H*W >= 2^31; everything else is bit-exact."""
        g = np.asarray(geoms, dtype=np.int32).reshape(-1, N.MRX_GEOM_INTS)
        pp = pack_polygons(g, class_ids, segms)
        rles = [[seg if isinstance(seg, dict) else {"size": [int(g[b, 0]), int(g[b, 1])],
                                                    "counts": b""} for seg in inst]
                for b, inst in enumerate(segms)]
        pk = pack_rle(g, class_ids, rles)   # a polygon instance: an empty string, not parsed
        return cls._decoded(lib, device, g, class_ids, pk, pp, stream)

    @classmethod
    def _decoded(cls, lib, device, g, class_ids, pk, pp, stream):
        """`from_rle` (pp None) and `from_coco`: the RLE tables of `pack_rle` and the polygon
        tables of `pack_polygons` in one upload; the RLE kernels write the planes of the RLE
        instances (all of them for `from_rle`), mrx_poly_decode those of the polygon ones."""
        torch = _torch()
        self = cls.__new__(cls)
        n, R, S = g.shape[0], pk["R"], pk["strings"].size
        status = np.zeros(n * R, np.int32)
        rle_extra = [status, pk["str_off"], pk["run_off"], pk["run_count"], pk["runs"],
                     pk["strings"]]
        poly = pp is not None and pp["P"] > 0
        run_rle = pp is None or bool(pp["rle"].any())
        if pp is not None:
            status[pp["poly"]] = N.MRX_RLE_ST_SKIP   # another path's plane: the decode skips it
        poly_extra = ([pp["vert"], pp["part_vert"], pp["part_inst"], pp["inst_part"],
                       pp["part_col"], pp["part_tog"]] if poly else [])

        def fill(layout, d_packed, d_off, d_status, d_str_off, d_run_off, d_run_count,
                 d_uploaded_runs, d_str, *d_poly):
            st = N.stream_ptr(stream)
            max_h, max_w = max(layout.max_h, 1), max(layout.max_w, 1)
            if run_rle:
                d_runs = torch.empty((max(S + pk["runs"].size, 1),), dtype=torch.int32,
                                     device=device)
                d_runs[S:S + pk["runs"].size].copy_(d_uploaded_runs)
                d_ends = torch.empty((d_runs.numel(),), dtype=torch.int64, device=device)
                if S:
                    N.check(lib.mrx_rle_parse(d_str, d_str_off, self.d_counts,
                                              d_runs, d_run_count, d_status, n,
                                              R, st), "mrx_rle_parse")
                N.check(lib.mrx_rle_decode(d_runs, d_run_off, d_run_count,
                                           d_ends, d_status, self.d_counts,
                                           self.d_geom, d_off, d_packed, n, R,
                                           max_h, max_w, st), "mrx_rle_decode")
            if poly:
                d_vert, d_part_vert, d_part_inst, d_inst_part, d_part_col, d_part_tog = d_poly
                n_col, n_tog = int(pp["part_col"][-1]), int(pp["part_tog"][-1])
                d_tog = torch.empty((max(n_tog, 1),), dtype=torch.int32, device=device)
                d_col_start = torch.empty((max(n_col, 1),), dtype=torch.int64, device=device)
                d_carry = torch.empty((max(n_col, 1),), dtype=torch.uint8, device=device)
                N.check(lib.mrx_poly_decode(
                    d_vert, d_part_vert, d_part_inst, d_part_col, d_part_tog, pp["P"], d_inst_part,
                    d_tog, d_col_start, d_carry, self.d_counts, self.d_geom, d_off, d_packed, n, R,
                    max_h, max_w, st), "mrx_poly_decode")

        d_status, *_ = self._stage(lib, device, g, class_ids, pk["counts"],
                                   rle_extra + poly_extra, fill, stream)
        with _stream_ctx(stream):
            status = d_status.cpu().numpy().reshape(n, R)     # the one synchronisation
            self.extents = self.planes.d_extents.cpu().numpy()
        if pp is not None:
            status = np.where(pp["poly"].reshape(n, R), 0, status)
        for b, k in zip(*np.nonzero(status)):
            what = [msg for bit, msg in _RLE_STATUS if status[b, k] & bit]
            hw = int(self.geom[b, 0]) * int(self.geom[b, 1])
            raise ValueError(f"image {b}, instance {k}: " + "; ".join(what).format(hw=hw))
        return self

    def _stage(self, lib, device, geoms, class_ids, counts, extra, fill, stream):
        """The one staging step of both constructors, once they have checked their input: the
        layout and the class-id table, one upload of every table (the fill's own arrays `extra`
        last), the packed slots, fill(layout, d_packed, d_off, *device views of extra) writing
        the planes, and mrx_mask_extents of every plane over its whole image.  Sets the
        attributes and `planes`; returns the device views of `extra`."""
        torch = _torch()
        n, R = geoms.shape[0], max(int(counts.max(initial=0)), 1)
        layout = BatchLayout(geoms, R, limits=False)
        self.n, self.R, self.geom, self.counts = n, R, layout.geom, counts
        regions = np.zeros((n, R, 4), dtype=np.int32)      # (0, 0, H_b, W_b): the whole image
        regions[:, :, 2:] = layout.geom[:, None, :2]
        tables = [layout.packed_off[:-1], counts, _class_id_table(class_ids, n, R), layout.geom,
                  regions, *extra]
        with _stream_ctx(stream):
            d_off, self.d_counts, self.d_class_ids, self.d_geom, d_regions, *d_extra = \
                _upload_parts(tables, device)
            d_packed = torch.empty((max(int(layout.packed_off[-1]), 1),), dtype=torch.uint8,
                                   device=device)
            fill(layout, d_packed, d_off, *d_extra)
            d_areas = torch.empty((n, R), dtype=torch.int64, device=device)
            d_ext = torch.empty((n, R, 4), dtype=torch.int32, device=device)
            N.check(lib.mrx_mask_extents(d_packed, d_off, self.d_counts,
                                         self.d_geom, d_regions, d_areas,
                                         d_ext, n, R, N.stream_ptr(stream)),
                    "mrx_mask_extents")
        self.planes = Planes(d_packed, d_off, self.d_counts, d_areas, d_ext, R)
        self.d_regions = d_regions
        return d_extra

    def boundary_planes(self, dilation_ratio=0.02, stream=None):
        """EXTENSION: `Planes` of the boundaries of this batch's masks, as boundary_iou_api's
        mask_to_boundary computes them for `dilation_ratio` (`boundary_dilation`), each over its
        whole image (mrx_mask_boundary, then mrx_mask_extents for the areas; the extents are the
        masks')."""
        d = boundary_dilation(self.geom, dilation_ratio)
        with _stream_ctx(stream):
            d_dil = _torch().from_numpy(d).to(self.d_geom.device)
            return mask_boundary_planes(N.load(), self.planes, self.d_geom, self.d_regions, d_dil,
                                        self.n, int(self.geom[:, 1].max(initial=1)), {}, stream)

    def set_counts(self, counts, stream=None):
        """Keep only the first counts[b] instances of each image (counts[b] <= M_b), as upstream
        cuts the ground truth to the rows `trim_zeros` leaves of its boxes."""
        counts = np.asarray(counts, dtype=np.int32).reshape(self.n)
        if (counts < 0).any() or (counts > self.counts).any():
            raise ValueError("counts must lie within the batch's instances")
        with _stream_ctx(stream):
            self.d_counts.copy_(_torch().from_numpy(counts))
        self.counts = counts


_RLE_STATUS = [
    (N.MRX_RLE_ST_CHAR, "a counts character outside '0'..'o'"),
    (N.MRX_RLE_ST_TRUNC, "the counts string ends inside a value"),
    (N.MRX_RLE_ST_RANGE, "a count is negative or does not fit in uint32"),
    (N.MRX_RLE_ST_SUM, "the counts do not sum to H*W = {hw}"),
]


def _class_id_table(class_ids, n, R):
    """int32 [n, R]: image b's class ids first, zeros after them."""
    cls = np.zeros((n, R), dtype=np.int32)
    for b, c in enumerate(class_ids):
        c = np.asarray(c)
        if c.size and (c.astype(np.int32) != c).any():
            raise ValueError(f"image {b}: class ids must be integers within int32")
        cls[b, :c.size] = c
    return cls


def pack_rle(geoms, class_ids, rles):
    """The host side of `MaskBatch.from_rle`, NumPy only: checks every instance and packs the
    batch into one byte buffer of strings and one uint32 array of uncompressed runs.  Instance
    i = b*R + k (R = max(1, max M_b)).  Returns a dict:
      counts     int32 [n]       M_b
      R          int
      strings    uint8 [S]       the compressed strings, instance i's at str_off[i]:str_off[i+1]
                                 (empty for uncompressed instances and k >= M_b)
      str_off    int64 [n*R+1]
      runs       uint32 [C]      the uncompressed runs, one instance after another
      run_off    int64 [n*R]     where instance i's runs are in the device buffer of
                                 [S parsed slots | runs]: str_off[i] for a string, S + its
                                 offset in `runs` for a list
      run_count  int32 [n*R]     len(runs of i) for a list, 0 otherwise (the parse writes it)"""
    g = np.asarray(geoms, dtype=np.int32).reshape(-1, N.MRX_GEOM_INTS)
    n = g.shape[0]
    if len(rles) != n or len(class_ids) != n:
        raise ValueError(f"{len(rles)} RLE lists and {len(class_ids)} class-id arrays for {n} "
                         "images")
    counts = np.zeros(n, dtype=np.int32)
    for b, (cls, inst) in enumerate(zip(class_ids, rles)):
        if np.shape(cls) != (len(inst),):
            raise ValueError(f"image {b}: {np.shape(cls)} class ids for {len(inst)} RLE dicts")
        counts[b] = len(inst)
    R = max(int(counts.max(initial=0)), 1)
    strings, runs = [], []
    str_len = np.zeros(n * R, np.int64)
    run_len = np.zeros(n * R, np.int64)
    is_list = np.zeros(n * R, bool)
    for b, inst in enumerate(rles):
        hw = [int(g[b, 0]), int(g[b, 1])]
        for k, rle in enumerate(inst):
            i, where = b * R + k, f"image {b}, instance {k}"
            try:
                size, c = rle["size"], rle["counts"]
            except (TypeError, KeyError):
                raise ValueError(f"{where}: an RLE is a dict with 'size' and 'counts'") from None
            got = [int(v) for v in np.ravel(size)]
            if got != hw:
                raise ValueError(f"{where}: size {got} is not the image's {hw}")
            if isinstance(c, str):
                try:
                    c = c.encode("ascii")
                except UnicodeEncodeError:
                    raise ValueError(f"{where}: the counts string is not ASCII") from None
            if isinstance(c, (bytes, bytearray)):
                strings.append(np.frombuffer(bytes(c), np.uint8))
                str_len[i] = len(c)
                continue
            a = np.asarray(c)
            if a.ndim != 1 or not (a.dtype.kind in "iu" or (a.size == 0 and a.dtype.kind == "f")):
                raise ValueError(f"{where}: counts must be bytes, str or a 1-D sequence of "
                                 f"integers, got {type(c).__name__}")
            if a.size and (a.min() < 0 or a.max() > 0xFFFFFFFF):
                raise ValueError(f"{where}: an uncompressed count is negative or does not fit in "
                                 "uint32")
            runs.append(a.astype(np.uint32))
            run_len[i] = a.size
            is_list[i] = True
    str_off = np.zeros(n * R + 1, np.int64)
    np.cumsum(str_len, out=str_off[1:])
    S = int(str_off[-1])
    list_off = np.concatenate([[0], np.cumsum(run_len)[:-1]]) if n * R else np.zeros(0, np.int64)
    run_off = np.where(is_list, S + list_off, str_off[:-1]).astype(np.int64)
    return {"counts": counts, "R": R,
            "strings": np.concatenate(strings) if strings else np.zeros(0, np.uint8),
            "str_off": str_off,
            "runs": np.concatenate(runs) if runs else np.zeros(0, np.uint32),
            "run_off": run_off, "run_count": np.where(is_list, run_len, 0).astype(np.int32)}


_INT_MIN, _INT_MAX = -(1 << 31), (1 << 31) - 1


def _polygon_parts(segm, where):
    """The parts of one polygon or box-list annotation as float64 [2V] coordinate arrays, each
    closed polygon as rleFrPoly receives it (`frPyObjects`' list dispatch on the first part's
    length; a box [x, y, w, h] becomes rleFrBbox's (x, y) (x, y+h) (x+w, y+h) (x+w, y))."""
    if len(segm) == 0:
        raise ValueError(f"{where}: an empty polygon list")
    parts = []
    for j, part in enumerate(segm):
        try:
            a = np.asarray(part, dtype=np.float64)
        except (TypeError, ValueError):
            raise ValueError(f"{where}: part {j} is not a list of numbers") from None
        if a.ndim != 1:
            raise ValueError(f"{where}: part {j} is not a flat list of numbers")
        parts.append(a)
    n0 = parts[0].size
    if n0 < 4:
        raise ValueError(f"{where}: the first part has {n0} numbers; a polygon needs more than "
                         "4 and a box exactly 4")
    if n0 == 4:
        if any(a.size != 4 for a in parts):
            raise ValueError(f"{where}: a box list (first part of 4 numbers) has a part that is "
                             "not 4 numbers")
        out = []
        for x, y, w, h in parts:
            xe, ye = x + w, y + h
            out.append(np.array([x, y, x, ye, xe, ye, xe, y]))
        return out
    for j, a in enumerate(parts):
        if a.size < 2:
            raise ValueError(f"{where}: part {j} has {a.size} numbers; a polygon part needs at "
                             "least one vertex")
    return [a[:a.size // 2 * 2] for a in parts]


def pack_polygons(geoms, class_ids, segms):
    """The host side of `MaskBatch.from_coco`'s polygons, NumPy only: checks every polygon or box
    list of segms (segms[b] a list of M_b COCO segmentations; RLE dicts are left to `pack_rle`)
    and lays the batch out for mrx_poly_decode.  Instance i = b*R + k (R = max(1, max M_b)).
    Each vertex coordinate c becomes rleFrPoly's (int)(5.0 * c + .5): NumPy's multiply, add and
    trunc round separately, as the C does.  Returns a dict:
      counts     int32 [n]       M_b
      R          int
      P          int             parts of every polygon instance, instance by instance
      poly       bool [n*R]      instance i is a polygon or box list
      rle        bool [n*R]      instance i is an RLE dict
      vert       int32 [V, 2]    the scaled vertices (x, y), part after part
      part_vert  int64 [P+1]     part p's vertices are vert[part_vert[p]:part_vert[p+1]]
      part_inst  int32 [P]       part p's instance i
      inst_part  int32 [n*R+1]   instance i's parts are inst_part[i]:inst_part[i+1]
      part_col   int64 [P+1]     part p's W_b + 1 column entries start at part_col[p]
      part_tog   int64 [P+1]     part p's toggle rows: part_tog[p]:part_tog[p+1], a bound of
                                 min(W_b, (|dx| + 2) // 5 + 1) + 1 per edge"""
    g = np.asarray(geoms, dtype=np.int32).reshape(-1, N.MRX_GEOM_INTS)
    n = g.shape[0]
    if len(segms) != n or len(class_ids) != n:
        raise ValueError(f"{len(segms)} segmentation lists and {len(class_ids)} class-id arrays "
                         f"for {n} images")
    counts = np.zeros(n, dtype=np.int32)
    for b, (cls, inst) in enumerate(zip(class_ids, segms)):
        if np.shape(cls) != (len(inst),):
            raise ValueError(f"image {b}: {np.shape(cls)} class ids for {len(inst)} "
                             "segmentations")
        counts[b] = len(inst)
    R = max(int(counts.max(initial=0)), 1)
    poly, rle = np.zeros(n * R, bool), np.zeros(n * R, bool)
    coords, part_inst = [], []
    inst_parts = np.zeros(n * R, np.int64)
    for b, inst in enumerate(segms):
        for k, segm in enumerate(inst):
            i, where = b * R + k, f"image {b}, instance {k}"
            if isinstance(segm, dict):
                rle[i] = True
                continue
            if not isinstance(segm, (list, tuple)):
                raise ValueError(f"{where}: a segmentation is a polygon list, a box list or an "
                                 f"RLE dict, got {type(segm).__name__}")
            poly[i] = True
            parts = _polygon_parts(segm, where)
            coords += parts
            part_inst += [i] * len(parts)
            inst_parts[i] = len(parts)
    # the numbers of every part at once: (int)(5.0 * c + .5), then the closed edges
    P = len(coords)
    part_inst = np.asarray(part_inst, np.int32)
    nv = np.array([a.size // 2 for a in coords], np.int64)
    part_vert = np.zeros(P + 1, np.int64)
    np.cumsum(nv, out=part_vert[1:])
    xy = np.concatenate(coords) if P else np.zeros(0)
    vpart = np.repeat(np.arange(P), nv)          # the part of each vertex

    def fail(bad_vertex, what):
        i = int(part_inst[vpart[int(np.flatnonzero(bad_vertex)[0])]])
        raise ValueError(f"image {i // R}, instance {i % R}: {what}")

    fin = np.isfinite(xy).reshape(-1, 2).all(1)
    if not fin.all():
        fail(~fin, "a coordinate is NaN or infinite")
    sc = np.trunc(np.add(np.multiply(5.0, xy), 0.5)).reshape(-1, 2)
    inr = ((sc >= _INT_MIN) & (sc <= _INT_MAX)).all(1)
    if not inr.all():
        fail(~inr, "a coordinate scaled by 5 does not fit in int")
    v = sc.astype(np.int64)
    nxt = np.arange(1, v.shape[0] + 1)
    nxt[part_vert[1:] - 1] = part_vert[:-1]      # the last vertex closes on the first
    d = np.abs(v[nxt] - v)
    ok = d.max(1, initial=0) <= _INT_MAX
    if not ok.all():
        fail(~ok, "two consecutive vertices scaled by 5 differ by more than int holds")
    W = g[part_inst // R, 1].astype(np.int64) if P else np.zeros(0, np.int64)
    edge_tog = np.minimum(W[vpart], (d[:, 0] + 2) // 5 + 1) + 1
    inst_part = np.zeros(n * R + 1, np.int64)
    np.cumsum(inst_parts, out=inst_part[1:])
    part_col, tog_off = np.zeros(P + 1, np.int64), np.zeros(P + 1, np.int64)
    np.cumsum(W + 1, out=part_col[1:])
    np.cumsum(np.add.reduceat(edge_tog, part_vert[:-1]) if P else edge_tog, out=tog_off[1:])
    verts = v.astype(np.int32)
    return {"counts": counts, "R": R, "P": P, "poly": poly, "rle": rle,
            "vert": verts, "part_vert": part_vert, "part_inst": part_inst,
            "inst_part": inst_part.astype(np.int32), "part_col": part_col, "part_tog": tog_off}


def mask_overlaps(lib, p1, p2, d_geom, n, stream=None):
    """mrx_mask_overlaps of two `Planes` of the same n images (d_geom [n, 8]): float32 device
    tensor [n, p1.R, p2.R], element (b, i, j) the IoU of mask i of p1 and mask j of p2 for i, j
    below the image's counts (the rest is not written)."""
    d_out = _torch().empty((n, p1.R, p2.R), dtype=_torch().float32, device=d_geom.device)
    N.check(lib.mrx_mask_overlaps(
        p1.d_packed, p1.d_packed_off, p1.d_counts, p1.d_areas, p1.d_extents, p1.R, p2.d_packed,
        p2.d_packed_off, p2.d_counts, p2.d_areas, p2.d_extents, p2.R, d_geom, d_out, n,
        N.stream_ptr(stream)), "mrx_mask_overlaps")
    return d_out


def comparison_threshold(t):
    """The float64 value compute_matches effectively compares its float32 IoUs with: NumPy (NEP 50)
    compares a Python float or int weakly, in float32, and a NumPy scalar strongly, in float64
    (`float32(0.7) < 0.7` is False, `float32(0.7) < np.float64(0.7)` is True)."""
    if isinstance(t, (np.generic, np.ndarray)):
        return float(t)
    if isinstance(t, (int, float)):
        return float(np.float32(t))
    raise TypeError(f"threshold must be a Python or NumPy real number, got {type(t).__name__}")


def mask_matches(lib, d_overlaps, d_pred_counts, d_pred_class_ids, d_scores, score_code, gt,
                 thresholds, score_threshold=0.0, stream=None):
    """mrx_mask_matches on overlaps [n, R1, gt.R] (see `mask_overlaps`), thresholds in launches of
    at most MRX_MAX_IOU_THRESHOLDS.  Returns device tensors (order [n, R1], pred_match
    [T, n, R1], gt_match [T, n, gt.R]) int32."""
    torch = _torch()
    n, R1, R2 = (int(v) for v in d_overlaps.shape)
    thr = [comparison_threshold(t) for t in thresholds]
    if not thr:
        raise ValueError("no IoU threshold given")
    dev = d_overlaps.device
    d_order = torch.empty((n, R1), dtype=torch.int32, device=dev)
    d_pm = torch.empty((len(thr), n, R1), dtype=torch.int32, device=dev)
    d_gm = torch.empty((len(thr), n, R2), dtype=torch.int32, device=dev)
    for t0 in range(0, len(thr), N.MRX_MAX_IOU_THRESHOLDS):
        chunk = thr[t0:t0 + N.MRX_MAX_IOU_THRESHOLDS]
        N.check(lib.mrx_mask_matches(
            d_overlaps, d_pred_counts, d_pred_class_ids, d_scores, score_code, gt.d_counts,
            gt.d_class_ids, N.double_array(chunk), len(chunk),
            comparison_threshold(score_threshold), d_order, d_pm[t0], d_gm[t0], n, R1, R2,
            N.stream_ptr(stream)), "mrx_mask_matches")
    return d_order, d_pm, d_gm


def coco_device_params(params):
    """(thresholds, area_rng, max_det) of a COCOeval-style params object (`iouThrs`, `areaRng`,
    `maxDets`) as the COCO kernels take them: the thresholds capped at 1 - 1e-10 as evaluateImg
    caps them, the area ranges flattened to [A * 2] float64, maxDets[-1].  Raises ValueError
    outside the kernels' limits."""
    return _device_params(params.iouThrs, params.areaRng, params.maxDets[-1], "maxDets[-1]")


def lvis_device_params(params):
    """`coco_device_params` of an LVISEval-style params object (`iou_thrs`, `area_rng`, and
    `max_dets` one int, the per-image cut)."""
    return _device_params(params.iou_thrs, params.area_rng, params.max_dets, "max_dets")


def _device_params(iou_thrs, area_rng, max_det, max_det_name):
    thr = [min(float(t), 1 - 1e-10) for t in np.ravel(iou_thrs)]
    rng = np.asarray(area_rng, dtype=np.float64).reshape(-1, 2)
    max_det = int(max_det)
    if not 1 <= len(thr) <= N.MRX_MAX_IOU_THRESHOLDS:
        raise ValueError(f"{len(thr)} IoU thresholds (need 1 to {N.MRX_MAX_IOU_THRESHOLDS})")
    if not 1 <= rng.shape[0] <= N.MRX_MAX_AREA_RANGES:
        raise ValueError(f"{rng.shape[0]} area ranges (need 1 to {N.MRX_MAX_AREA_RANGES})")
    if max_det < 1:
        raise ValueError(f"{max_det_name} = {max_det} (need >= 1)")
    return thr, rng.reshape(-1).tolist(), max_det


def coco_evaluate_batch(lib, pred, pred_class_ids, pred_scores, gt, gt_crowd, gt_area, class_map,
                        params, stream=None, status=None):
    """The per-image half of COCOeval (iouType "segm") for one batch: mrx_coco_ranks,
    mrx_coco_ious and mrx_coco_match, then one download and one synchronisation.  With `status`
    it is lvis-api's LVISEval (iouType "segm"): mrx_lvis_ranks (the per-image cut at
    `params.max_dets` and the federated filter) takes mrx_coco_ranks' place.

    pred: `Planes` of the predictions (areas and extents from mrx_mask_extents) of gt's images,
    pred_class_ids [n, pred.R] int32 and pred_scores [n, pred.R] float32 / float64 device tensors;
    gt: a `MaskBatch` whose class ids are dense category indices; gt_crowd [n, gt.R] (iscrowd;
    LVISEval passes zeros) and gt_area [n, gt.R] (the annotations' areas, float64) host arrays;
    class_map [C] int32 host array, prediction class id -> dense category or -1 (not evaluated);
    params: COCOeval's `iouThrs`, `areaRng`, `maxDets` (`coco_device_params`), or with status
    LVISEval's `iou_thrs`, `area_rng`, `max_dets` (`lvis_device_params`); status: None, or an
    [n, K] uint8 host array of MRX_LVIS_* bits per (image, dense category), uploaded in the one
    copy of the ground-truth tables (class_map's categories must then be < K; one at or above K
    is not evaluated).

    Returns a dict of host arrays: `counts` [n]; per prediction [n, pred.R] `cat`, `rank` (in
    its (image, category), in score order), `keep` (cat >= 0 and rank < maxDets[-1], and within
    the count; with status, mrx_lvis_ranks' rule), `area` (int64 pixels), `score` (float64);
    `match` [A, T, n, pred.R] int32 (the ground-truth index or -1) and `ignore` [A, T, n, pred.R]
    bool, defined where `keep` is (with status, without LVISEval's not-exhaustive rule, which is
    the caller's); and `d_iou`, the float64 device tensor [n, pred.R, gt.R] of mrx_coco_ious."""
    n, R1, R2 = gt.n, int(pred.R), int(gt.R)
    class_map = _coco_class_map(class_map)
    with _stream_ctx(stream):
        d_crowd, d_area, d_map, *d_status = _upload_parts(
            [np.ascontiguousarray(gt_crowd, dtype=np.uint8).reshape(n, R2),
             np.ascontiguousarray(gt_area, dtype=np.float64).reshape(n, R2), class_map]
            + _status_part(status, n), gt.d_geom.device)

        def ious(v, d_iou, st):
            v["area"].copy_(pred.d_areas.view(-1)[:n * R1].view(n, R1))
            N.check(lib.mrx_coco_ious(
                pred.d_packed, pred.d_packed_off, pred.d_counts, pred.d_areas, pred.d_extents,
                v["cat"], v["keep"], R1, gt.planes.d_packed, gt.planes.d_packed_off,
                gt.planes.d_counts, gt.planes.d_areas, gt.planes.d_extents, gt.d_class_ids,
                d_crowd, R2, gt.d_geom, d_iou, n, st), "mrx_coco_ious")

        return _coco_evaluate(lib, n, R1, R2, pred.d_counts, pred_class_ids, pred_scores,
                              gt.d_counts, gt.d_class_ids, d_crowd, d_area, d_map,
                              _scorer_params(params, status), np.int64, ious, stream, *d_status)


def _scorer_params(params, status):
    """The device parameters of COCOeval's params, or of LVISEval's when there is a status
    table."""
    return (coco_device_params if status is None else lvis_device_params)(params)


def _status_part(status, n):
    """[status as a C-contiguous uint8 [n, K] array] for the one upload, or [] without one."""
    if status is None:
        return []
    status = np.ascontiguousarray(status, dtype=np.uint8)
    if status.ndim != 2 or status.shape[0] != n or status.shape[1] < 1:
        raise ValueError(f"status must be [{n}, K >= 1], got {status.shape}")
    return [status]


def coco_box_evaluate_batch(lib, pred_boxes, pred_counts, pred_class_ids, pred_scores, gt_counts,
                            gt_cat, gt_boxes, gt_crowd, gt_area, class_map, params, stream=None,
                            status=None):
    """The per-image half of COCOeval (iouType "bbox") for one batch of n images: mrx_coco_ranks
    (mrx_lvis_ranks with `status`: LVISEval "bbox"), mrx_coco_box_ious and
    mrx_coco_match_f64area, then one download and one synchronisation.  No mask is read.

    pred_boxes [n, R1, 4]: int32 (y1, x1, y2, x2), the kept boxes of mrx_unmold_prepare (their
    `bbox` is [x1, y1, x2 - x1, y2 - y1]), or float64 [x, y, w, h], results' `bbox`;
    pred_counts [n] int32, pred_class_ids [n, R1] int32 and pred_scores [n, R1] float32 /
    float64.  Each of those is a device tensor or a host array; the host arrays go up in one copy
    with the ground truth.  gt_counts [n], gt_cat [n, R2] (dense category indices), gt_boxes
    [n, R2, 4] float64 [x, y, w, h], gt_crowd [n, R2] and gt_area [n, R2] host arrays; class_map,
    params and status as for `coco_evaluate_batch`.

    Returns `coco_evaluate_batch`'s dict, with `area` float64 (each kept prediction's w*h, as
    loadRes stores it for a bbox result) and `d_iou` from mrx_coco_box_ious."""
    torch = _torch()
    gt_cat = np.ascontiguousarray(gt_cat, dtype=np.int32)
    n, R2 = gt_cat.shape
    R1 = int(pred_boxes.shape[1])
    class_map = _coco_class_map(class_map)
    pred = [pred_boxes, pred_counts, pred_class_ids, pred_scores]
    dev = next((x.device for x in pred if not isinstance(x, np.ndarray)),
               torch.device("cuda", torch.cuda.current_device()))
    parts = [np.ascontiguousarray(gt_counts, dtype=np.int32).reshape(n), gt_cat,
             np.ascontiguousarray(gt_boxes, dtype=np.float64).reshape(n, R2, 4),
             np.ascontiguousarray(gt_crowd, dtype=np.uint8).reshape(n, R2),
             np.ascontiguousarray(gt_area, dtype=np.float64).reshape(n, R2), class_map]
    parts += _status_part(status, n)
    on_host = [k for k, x in enumerate(pred) if isinstance(x, np.ndarray)]
    with _stream_ctx(stream):
        up = _upload_parts(parts + [np.ascontiguousarray(pred[k]) for k in on_host], dev)
        d_counts, d_cat, d_boxes, d_crowd, d_area, d_map = up[:6]
        d_status = up[6:len(parts)]
        for k, t in zip(on_host, up[len(parts):]):
            pred[k] = t
        pred_boxes, pred_counts, pred_class_ids, pred_scores = pred
        form = {torch.int32: N.MRX_BOX_YXYX_I32, torch.float64: N.MRX_BOX_XYWH_F64}[
            pred_boxes.dtype]

        def ious(v, d_iou, st):
            N.check(lib.mrx_coco_box_ious(
                pred_boxes, form, pred_counts, v["cat"], v["keep"], R1, d_boxes, d_counts, d_cat,
                d_crowd, R2, v["area"], d_iou, n, st), "mrx_coco_box_ious")

        return _coco_evaluate(lib, n, R1, R2, pred_counts, pred_class_ids, pred_scores, d_counts,
                              d_cat, d_crowd, d_area, d_map, _scorer_params(params, status),
                              np.float64, ious, stream,
                              *d_status)


def check_dilation_ratio(dilation_ratio):
    """dilation_ratio as a float: a finite real number > 0, else ValueError."""
    ok = isinstance(dilation_ratio, (int, float, np.integer, np.floating)) and \
        not isinstance(dilation_ratio, (bool, np.bool_))
    r = float(dilation_ratio) if ok else math.nan
    if not (math.isfinite(r) and r > 0):
        raise ValueError(f"dilation_ratio must be a finite number > 0, got {dilation_ratio!r}")
    return r


def boundary_dilation(geoms, dilation_ratio):
    """int32 [n]: boundary_iou_api's dilation of each image of `geoms` ([n, 8], see make_geom),
    max(1, int(round(dilation_ratio * sqrt(H**2 + W**2)))) with Python's round (half to even).
    Values above 2^30 are stored as 2^30: any d at or above an image side erodes everything."""
    r = check_dilation_ratio(dilation_ratio)
    g = np.asarray(geoms, dtype=np.int64).reshape(-1, N.MRX_GEOM_INTS)
    return np.array([min(max(1, int(round(r * math.sqrt(int(H) ** 2 + int(W) ** 2)))), 1 << 30)
                     for H, W in g[:, :2]], dtype=np.int32).reshape(-1)


def mask_boundary_planes(lib, planes, d_geom, d_regions, d_dilation, n, max_w, bufs, stream=None,
                         name="boundary"):
    """`Planes` of the boundaries of `planes` (n images, d_geom [n, 8]): mrx_mask_boundary with
    regions d_regions [n, planes.R, 4] and dilations d_dilation [n] int32 into a buffer of the
    same slot layout, then mrx_mask_extents over it with the same regions for the areas.  The
    boundary planes, areas and (the masks') extents are kept in `bufs` under `name`."""
    torch = _torch()
    R, dev = int(planes.R), d_geom.device
    d_bnd = _buffer(bufs, name + "_packed", planes.d_packed.numel(), torch.uint8, dev)
    d_areas = _buffer(bufs, name + "_areas", n * R, torch.int64, dev)
    d_ext = _buffer(bufs, name + "_extents", n * R * 4, torch.int32, dev)
    st = N.stream_ptr(stream)
    N.check(lib.mrx_mask_boundary(
        planes.d_packed, planes.d_packed_off, planes.d_counts, d_geom, d_regions, d_dilation,
        d_bnd, n, R, max(int(max_w), 1), st),
        "mrx_mask_boundary")
    N.check(lib.mrx_mask_extents(
        d_bnd, planes.d_packed_off, planes.d_counts, d_geom, d_regions, d_areas, d_ext, n, R,
        st), "mrx_mask_extents")
    return Planes(d_bnd, planes.d_packed_off, planes.d_counts, d_areas[:n * R].view(n, R),
                  d_ext[:n * R * 4].view(n, R, 4), R)


def coco_boundary_evaluate_batch(lib, pred, pred_regions, pred_class_ids, pred_scores, gt,
                                 gt_crowd, gt_area, class_map, params, dilation_ratio=0.02,
                                 stream=None, bufs=None):
    """The per-image half of COCOeval for iouType "boundary" (boundary_iou_api) for one batch:
    mrx_coco_ranks, the boundaries of both sides (`mask_boundary_planes`: the predictions inside
    pred_regions [n, pred.R, 4] int32, e.g. their boxes, the ground truth over its whole images),
    mrx_coco_boundary_ious and mrx_coco_match, then one download and one synchronisation.  The
    per-image dilations (`boundary_dilation`) go up in the one copy of the ground-truth tables.
    Arguments and result as for `coco_evaluate_batch` (`area` is the mask's pixel count); `bufs`
    keeps the boundary buffers between calls."""
    n, R1, R2 = gt.n, int(pred.R), int(gt.R)
    class_map = _coco_class_map(class_map)
    dil = boundary_dilation(gt.geom, dilation_ratio)
    max_w = int(gt.geom[:, 1].max(initial=1))
    bufs = {} if bufs is None else bufs
    with _stream_ctx(stream):
        d_crowd, d_area, d_map, d_dil = _upload_parts(
            [np.ascontiguousarray(gt_crowd, dtype=np.uint8).reshape(n, R2),
             np.ascontiguousarray(gt_area, dtype=np.float64).reshape(n, R2), class_map, dil],
            gt.d_geom.device)

        def ious(v, d_iou, st):
            v["area"].copy_(pred.d_areas.view(-1)[:n * R1].view(n, R1))
            bp = mask_boundary_planes(lib, pred, gt.d_geom, pred_regions, d_dil, n, max_w, bufs,
                                      stream, "pred_boundary")
            bg = mask_boundary_planes(lib, gt.planes, gt.d_geom, gt.d_regions, d_dil, n, max_w,
                                      bufs, stream, "gt_boundary")
            N.check(lib.mrx_coco_boundary_ious(
                pred.d_packed, pred.d_packed_off, pred.d_counts, pred.d_areas, pred.d_extents,
                bp.d_packed, bp.d_areas, v["cat"], v["keep"], R1, gt.planes.d_packed,
                gt.planes.d_packed_off, gt.planes.d_counts, gt.planes.d_areas,
                gt.planes.d_extents, bg.d_packed, bg.d_areas, gt.d_class_ids, d_crowd, R2,
                gt.d_geom, d_iou, n, st), "mrx_coco_boundary_ious")

        return _coco_evaluate(lib, n, R1, R2, pred.d_counts, pred_class_ids, pred_scores,
                              gt.d_counts, gt.d_class_ids, d_crowd, d_area, d_map,
                              coco_device_params(params), np.int64, ious, stream)


def _coco_class_map(class_map):
    class_map = np.asarray(class_map, dtype=np.int32).reshape(-1)
    return class_map if class_map.size else np.full(1, -1, np.int32)


def _coco_evaluate(lib, n, R1, R2, d_pred_counts, pred_class_ids, pred_scores, d_gt_counts,
                   d_gt_cat, d_crowd, d_area, d_map, dparams, area_dtype, ious, stream,
                   d_status=None):
    """What every IoU type shares, on the current stream: the rank step (mrx_coco_ranks, or
    mrx_lvis_ranks with the [n, K] status table d_status), `ious(v, d_iou, st)` (fills d_iou
    [n, R1, R2] and the predictions' `area` in the output views v), the match kernel for
    area_dtype (int64 mask pixels or float64 box areas), then the one download of the output
    buffer and its one synchronisation.  dparams: (thresholds, area_rng, max_det) of
    `coco_device_params` / `lvis_device_params`.  Returns `coco_evaluate_batch`'s dict."""
    torch = _torch()
    thr, rng, max_det = dparams
    T, A = len(thr), len(rng) // 2
    dev = d_map.device
    score_code = {torch.float32: N.MRX_F32, torch.float64: N.MRX_F64}[pred_scores.dtype]
    st = N.stream_ptr(stream)
    # everything that comes back lives in one device buffer laid out by _part_offsets
    parts = {"counts": ((n,), np.int32), "cat": ((n, R1), np.int32), "rank": ((n, R1), np.int32),
             "keep": ((n, R1), np.uint8), "area": ((n, R1), area_dtype),
             "score": ((n, R1), np.float64), "match": ((A, T, n, R1), np.int32),
             "ignore": ((A, T, n, R1), np.uint8)}
    specs = list(parts.values())
    d_out = torch.empty((max(int(_part_offsets(specs)[-1]), 16),), dtype=torch.uint8, device=dev)
    v = dict(zip(parts, _part_views(d_out, specs)))
    d_walk = torch.empty((n, R1), dtype=torch.int32, device=dev)
    d_iou = torch.empty((n, R1, R2), dtype=torch.float64, device=dev)
    v["counts"].copy_(d_pred_counts[:n])
    v["score"].copy_(pred_scores[:n])
    if d_status is None:
        N.check(lib.mrx_coco_ranks(
            pred_class_ids, pred_scores, score_code, d_pred_counts, d_map, int(d_map.numel()),
            max_det, v["cat"], v["rank"], v["keep"], d_walk, n, R1, st), "mrx_coco_ranks")
    else:
        N.check(lib.mrx_lvis_ranks(
            pred_class_ids, pred_scores, score_code, d_pred_counts, d_map, int(d_map.numel()),
            d_status, int(d_status.shape[1]), max_det, v["cat"], v["rank"], v["keep"], d_walk, n,
            R1, st), "mrx_lvis_ranks")
    ious(v, d_iou, st)
    match = {np.dtype(np.int64): "mrx_coco_match",
             np.dtype(np.float64): "mrx_coco_match_f64area"}[np.dtype(area_dtype)]
    N.check(getattr(lib, match)(
        d_iou, d_pred_counts, v["cat"], v["keep"], d_walk, v["area"], d_gt_counts, d_gt_cat,
        d_crowd, d_area, N.double_array(thr), T, N.double_array(rng), A, v["match"], v["ignore"],
        n, R1, R2, st), match)
    host = d_out.cpu().numpy()         # the one synchronisation
    out = dict(zip(parts, _part_views(host, specs)))
    out["keep"] = (out["keep"] != 0) & (np.arange(R1)[None, :] < out["counts"][:, None])
    out["ignore"] = out["ignore"] != 0
    out["d_iou"] = d_iou
    return out


def trace_packed_contours(lib, device, d_packed, d_packed_off, d_counts, d_geom, d_regions, layout,
                          stream=None, bufs=None):
    """mrx_contours_count, one host read of the segment counts, mrx_contours_write, over the planes
    of a BatchLayout as mrx_pack_masks writes them; d_regions [n,R,4] int32 pixel rectangles; `bufs`
    keeps the work and output buffers between calls.  Returns (d_vertices [V,2] float32,
    d_contour_off [C+1] int64, inst_contour_off int64 ndarray [n*R+1])."""
    with _stream_ctx(stream):
        return _trace_packed_contours(lib, device, d_packed, d_packed_off, d_counts, d_geom,
                                      d_regions, layout, stream, {} if bufs is None else bufs)


def _stream_ctx(stream):
    """Make `stream` current (host reads then wait for the work queued on it)."""
    import contextlib

    return contextlib.nullcontext() if stream is None else _torch().cuda.stream(stream)


def _trace_packed_contours(lib, device, d_packed, d_packed_off, d_counts, d_geom, d_regions,
                           layout, stream, bufs):
    torch = _torch()
    st = N.stream_ptr(stream)
    n, R, max_h = layout.n, layout.R, layout.max_h
    ni = n * R
    d_rows = _buffer(bufs, "rows", ni * (max_h + 1), torch.int32, device)
    d_inst = _buffer(bufs, "inst", ni + 1, torch.int64, device)
    args = (d_packed, d_packed_off, d_counts, d_geom, d_regions, d_rows, d_inst)
    N.check(lib.mrx_contours_count(*args, n, R, max_h, st), "mrx_contours_count")
    seg_off = d_inst[:ni + 1].cpu().numpy()     # how many segments: sizes every output
    S = int(seg_off[-1])
    smax = int(np.diff(seg_off).max()) if ni else 0
    if S > N.MRX_MAX_CONTOUR_SEGMENTS:
        raise N.MrxError(f"{S} contour segments in one batch (limit {N.MRX_MAX_CONTOUR_SEGMENTS}); "
                         "split the batch")
    d_scr = _buffer(bufs, "scratch", N.contour_scratch_bytes(S), torch.uint8, device)
    d_vert = _buffer(bufs, "vertices", 2 * (S + S // 4), torch.float32, device)
    d_coff = _buffer(bufs, "contour_off", S // 4 + 1, torch.int64, device)
    d_icoff = _buffer(bufs, "inst_contour_off", ni + 1, torch.int64, device)
    N.check(lib.mrx_contours_write(*args, S, smax, d_scr, d_vert, d_coff, d_icoff, n, R, max_h,
                                   st),
            "mrx_contours_write")
    icoff = d_icoff[:ni + 1].cpu().numpy()
    n_contours = int(icoff[-1])
    # every contour repeats its first vertex: V = S + C
    return d_vert[:2 * (S + n_contours)].view(-1, 2), d_coff[:n_contours + 1], icoff


def _download_contours(d_vert, d_coff):
    """Host copies (float64 vertices [V, 2], int64 contour offsets) of a trace's output."""
    return d_vert.cpu().numpy().astype(np.float64), d_coff.cpu().numpy()


def contours_to_lists(verts, contour_off, inst_contour_off, counts, layout):
    """Per image b, per kept instance k < counts[b], the list of float64 [V, 2] polygons: contour
    c of instance i (`layout.kept_instances`) for c in [inst_contour_off[i], inst_contour_off[i+1])
    has the vertices verts[contour_off[c]:contour_off[c+1]]."""
    polys = np.split(verts, contour_off[1:-1]) if len(contour_off) > 1 else []
    out = [[] for _ in counts]
    for b, _, i in layout.kept_instances(counts):
        out[b].append(polys[int(inst_contour_off[i]):int(inst_contour_off[i + 1])])
    return out


class AnchorGenerator:
    """`get_anchors` on the device; memoised by image shape like upstream's method."""

    def __init__(self, config, device=None):
        N.require_cuda()
        torch = _torch()
        self.lib = N.load()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None \
            else torch.device(device)
        self.scales = [float(s) for s in config.RPN_ANCHOR_SCALES]
        self.ratios = [float(r) for r in config.RPN_ANCHOR_RATIOS]
        self.strides = [int(s) for s in config.BACKBONE_STRIDES]
        self.anchor_stride = int(config.RPN_ANCHOR_STRIDE)
        if len(self.scales) != len(self.strides):
            raise ValueError("RPN_ANCHOR_SCALES and BACKBONE_STRIDES must have equal length")
        self._cache = {}

    def count(self, image_shape):
        out = C.c_longlong(0)
        N.check(self.lib.mrx_anchor_count(
            int(image_shape[0]), int(image_shape[1]), N.int_array(self.strides),
            len(self.strides), len(self.ratios), self.anchor_stride, C.byref(out)),
            "mrx_anchor_count")
        return int(out.value)

    def generate_device(self, image_shape, out=None, stream=None):
        """[A,4] float32 device tensor (not cached)."""
        torch = _torch()
        A = self.count(image_shape)
        if out is None:
            out = torch.empty((A, 4), dtype=torch.float32, device=self.device)
        N.check(self.lib.mrx_anchors(
            out, int(image_shape[0]), int(image_shape[1]),
            N.double_array(self.scales), N.double_array(self.ratios),
            N.int_array(self.strides), len(self.strides), len(self.ratios),
            self.anchor_stride, N.stream_ptr(stream)), "mrx_anchors")
        return out

    def get_anchors(self, image_shape):
        key = tuple(int(v) for v in image_shape)
        if key not in self._cache:
            self._cache[key] = self.generate_device(image_shape).cpu().numpy()
        return self._cache[key]


def resize_image_geometry(h, w, min_dim, max_dim, min_scale, mode):
    """Host-side scalar logic of upstream utils.resize_image (serve.py:91-97): returns
    (new_h, new_w, top, left, out_h, out_w, window, scale, padding).  `crop` mode is
    random/training-only and not part of serving."""
    scale = 1
    if mode == "none":
        return h, w, 0, 0, h, w, (0, 0, h, w), 1, [(0, 0), (0, 0), (0, 0)]
    if min_dim:
        scale = max(1, min_dim / min(h, w))
    if min_scale and scale < min_scale:
        scale = min_scale
    if max_dim and mode == "square":
        image_max = max(h, w)
        if round(image_max * scale) > max_dim:
            scale = max_dim / image_max
    nh, nw = (round(h * scale), round(w * scale)) if scale != 1 else (h, w)
    if mode == "square":
        top = (max_dim - nh) // 2
        bottom = max_dim - nh - top
        left = (max_dim - nw) // 2
        right = max_dim - nw - left
        out_h, out_w = max_dim, max_dim
    elif mode == "pad64":
        assert min_dim % 64 == 0, "Minimum dimension must be a multiple of 64"
        if nh % 64 > 0:
            max_h = nh - (nh % 64) + 64
            top = (max_h - nh) // 2
            bottom = max_h - nh - top
        else:
            top = bottom = 0
        if nw % 64 > 0:
            max_w = nw - (nw % 64) + 64
            left = (max_w - nw) // 2
            right = max_w - nw - left
        else:
            left = right = 0
        out_h, out_w = nh + top + bottom, nw + left + right
    else:
        raise Exception("Mode {} not supported".format(mode))
    if top < 0 or left < 0:
        raise ValueError("image larger than IMAGE_MAX_DIM after scaling")
    padding = [(top, bottom), (left, right), (0, 0)]
    window = (top, left, nh + top, nw + left)
    return nh, nw, top, left, out_h, out_w, window, scale, padding


class Molder:
    """cv2.resize + resize_image + mold_image on the device (serve.py:88-98)."""

    def __init__(self, config, device=None):
        N.require_cuda()
        torch = _torch()
        self.lib = N.load()
        self.config = config
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None \
            else torch.device(device)

    def cv2_resize_device(self, d_img, size_hw, stream=None):
        torch = _torch()
        sh, sw = int(d_img.shape[0]), int(d_img.shape[1])
        dh, dw = int(size_hw[0]), int(size_hw[1])
        out = torch.empty((dh, dw, 3), dtype=torch.uint8, device=self.device)
        N.check(self.lib.mrx_cv2_resize_u8c3(d_img, sh, sw, out, dh, dw,
                                             N.stream_ptr(stream)), "mrx_cv2_resize_u8c3")
        return out

    def mold_device(self, d_img, out_dtype=np.float32, want_u8=False, stream=None):
        """resize_image + mold_image for a uint8 HxWx3 device image.
        Returns (molded, molded_u8|None, window, scale, padding)."""
        torch = _torch()
        cfg = self.config
        h, w = int(d_img.shape[0]), int(d_img.shape[1])
        nh, nw, top, left, oh, ow, window, scale, padding = resize_image_geometry(
            h, w, cfg.IMAGE_MIN_DIM, cfg.IMAGE_MAX_DIM, cfg.IMAGE_MIN_SCALE,
            cfg.IMAGE_RESIZE_MODE)
        out = torch.empty((oh, ow, 3), dtype=_torch_dtype(out_dtype), device=self.device)
        u8 = torch.empty((oh, ow, 3), dtype=torch.uint8, device=self.device) if want_u8 \
            else None
        mean = [float(v) for v in np.asarray(cfg.MEAN_PIXEL, dtype=np.float64)]
        N.check(self.lib.mrx_mold_image(
            d_img, h, w, nh, nw, top, left, oh, ow, N.double_array(mean),
            _dtype_code(out_dtype), out, u8, N.stream_ptr(stream)),
            "mrx_mold_image")
        return out, u8, window, scale, padding


    # ------------------------------------------------------------------ JPEG (csrc/jpeg.cu)
    def _jpeg_buffer(self, name, n, dtype):
        """The decoder's reusable device buffers, grown when a batch needs more."""
        torch = _torch()
        bufs = self.__dict__.setdefault("_jpeg_bufs", {})
        t = bufs.get(name)
        if t is None or t.numel() < n:
            t = bufs[name] = torch.empty((max(int(n), 1),), dtype=dtype, device=self.device)
        return t

    def _jpeg_upload(self, plan):
        """The batch's one upload: desc, unit -> image table, tables and files in one pinned
        buffer and one H2D copy.  Returns device views (desc, unit_img, tabs, files)."""
        torch = _torch()
        parts = [plan.desc.view(np.uint8).reshape(-1), plan.unit_img.view(np.uint8),
                 plan.tabs.reshape(-1), plan.files]
        off = _slot_offsets(np.asarray([p.size for p in parts], dtype=np.int64), 16)
        total = int(off[-1])
        if getattr(self, "_h_jpeg", None) is None or self._h_jpeg.numel() < total:
            self._h_jpeg = torch.empty((total,), dtype=torch.uint8).pin_memory()
        hs = self._h_jpeg.numpy()
        for p, o in zip(parts, off[:-1]):
            hs[int(o):int(o) + p.size] = p
        d = self._jpeg_buffer("upload", total, torch.uint8)
        d[:total].copy_(self._h_jpeg[:total], non_blocking=True)
        views = [d[int(o):int(o) + p.size] for p, o in zip(parts, off[:-1])]
        return views[0].view(torch.int64), views[1].view(torch.int32), views[2], views[3]

    def jpeg_coefficients(self, plan, stream=None):
        """Enqueue `mrx_jpeg_coefficients` for a `jpeg.Plan`: returns (d_coef int16 [blocks, 64]
        in decode order, d_status [B] int32, the device upload).  Nothing is synchronised."""
        torch = _torch()
        d_desc, d_unit_img, d_tabs, d_files = up = self._jpeg_upload(plan)
        d_unst = self._jpeg_buffer("unst", plan.unst_bytes, torch.uint8)
        d_work = self._jpeg_buffer("work", plan.work_words, torch.int32)
        d_coef = self._jpeg_buffer("coef", plan.coef_blocks * 64, torch.int16)
        d_status = self._jpeg_buffer("status", plan.B, torch.int32)
        N.check(self.lib.mrx_jpeg_coefficients(
            d_files, d_desc, d_tabs, d_unit_img, plan.B,
            max(plan.units, 1), plan.S, plan.max_subs, d_unst, d_work, d_coef,
            plan.coef_blocks, d_status, N.stream_ptr(stream)), "mrx_jpeg_coefficients")
        return d_coef[:plan.coef_blocks * 64].view(-1, 64), d_status[:plan.B], up

    def jpeg_decode_into(self, plan, d_out, out_off, stream=None):
        """Enqueue the decode of every file of `plan` into the uint8 slots d_out + out_off[b]
        (int64 byte offsets; image b is plan.shapes[b]).  Returns d_status [B] (device); call
        `jpeg_check` on it once the work that reads the slots has been enqueued."""
        torch = _torch()
        d_coef, d_status, (d_desc, _, d_tabs, _) = self.jpeg_coefficients(plan, stream)
        d_planes = self._jpeg_buffer("planes", plan.plane_bytes, torch.uint8)
        d_off = torch.from_numpy(np.ascontiguousarray(out_off, dtype=np.int64)).to(
            self.device, non_blocking=True)
        N.check(self.lib.mrx_jpeg_pixels(
            d_desc, d_tabs, d_coef, d_status, plan.B, plan.max_blocks,
            plan.max_pixels, d_planes, d_out, d_off, N.stream_ptr(stream)),
            "mrx_jpeg_pixels")
        return d_status

    @staticmethod
    def jpeg_check(d_status, index=None):
        """Download the status words (the one synchronisation) and raise ValueError naming the
        first image whose entropy-coded data was corrupt.  index[b]: the caller's index of b."""
        from . import jpeg

        st = d_status.cpu().numpy()
        for b in np.flatnonzero(st):
            i = int(index[b]) if index is not None else int(b)
            raise jpeg.JpegError(f"image {i}: corrupt JPEG data ({jpeg.status_reasons(st[b])})")

    def decode_jpeg_batch(self, blobs, S=None, stream=None):
        """uint8 [H, W, 3] RGB CUDA tensors, one per JPEG file: cv2.imdecode + BGR2RGB bit for
        bit.  The images share one buffer; equal sizes make them one contiguous [B, H, W, 3]."""
        from . import jpeg

        torch = _torch()
        plan = jpeg.Plan(blobs, jpeg.DEFAULT_S if S is None else S)
        if plan.B == 0:
            return []
        sizes = np.asarray([h * w * 3 for h, w, _ in plan.shapes], dtype=np.int64)
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        out = torch.empty((int(off[-1]),), dtype=torch.uint8, device=self.device)
        self.jpeg_check(self.jpeg_decode_into(plan, out, off[:-1], stream))
        return [out[int(off[b]):int(off[b + 1])].view(plan.shapes[b]) for b in range(plan.B)]

    # ------------------------------------------------------------------ batched (one launch each)
    def stage_images(self, images, align=16, stream=None):
        """Every image in its slot of one device buffer: uint8 HxWx3 NumPy images through one
        pinned staging buffer and one H2D copy, JPEG files (bytes) decoded on the device into
        their slots.  Returns (d_src, off [B+1] int64 slot offsets, shapes, d_status or None,
        jidx: the indices of the JPEG items).  Call `jpeg_check(d_status, jidx)` once the work
        that reads the slots has been enqueued."""
        from . import jpeg

        torch = _torch()
        B = len(images)
        is_jpeg = [isinstance(im, (bytes, bytearray, memoryview)) for im in images]
        jidx = [b for b in range(B) if is_jpeg[b]]
        plan = jpeg.Plan([images[b] for b in jidx], index=jidx) if jidx else None
        shapes = [None] * B
        for k, b in enumerate(jidx):
            shapes[b] = plan.shapes[k]
        for b in range(B):
            if shapes[b] is None:
                shapes[b] = tuple(int(v) for v in images[b].shape)
        sizes = [sh[0] * sh[1] * 3 for sh in shapes]
        off = _slot_offsets(np.asarray(sizes, dtype=np.int64), align)
        total = int(off[-1])
        if getattr(self, "_h_stage", None) is None or self._h_stage.numel() < total:
            self._h_stage = torch.empty((total,), dtype=torch.uint8).pin_memory()
        hs = self._h_stage.numpy()
        for b, im in enumerate(images):
            if not is_jpeg[b]:
                hs[int(off[b]):int(off[b]) + sizes[b]] = np.ascontiguousarray(im).reshape(-1)
        d_src = self._h_stage[:total].to(self.device, non_blocking=True)
        d_status = self.jpeg_decode_into(plan, d_src, off[jidx], stream) if jidx else None
        return d_src, off, shapes, d_status, jidx

    # ------------------------------------------------------------------ batched (one launch each)
    def cv2_resize_batch_device(self, images, size_hw, stream=None, return_sources=False):
        """`cv2.resize(img, (S, S))` for a list of images of ANY sizes in one launch: uint8 HxWx3
        NumPy images or JPEG files as bytes, staged by `stage_images` (JPEG files decoded on the
        device into their slots).  Returns uint8 [B, dh, dw, 3] on the device; with
        return_sources also each image's pixels for later steps: the array itself, or for a JPEG
        file its decoded slot (uint8 [H, W, 3] on the device)."""
        torch = _torch()
        B = len(images)
        dh, dw = int(size_hw[0]), int(size_hw[1])
        d_src, off, shapes, d_status, jidx = self.stage_images(images, 16, stream)
        hw = np.asarray([sh[:2] for sh in shapes], dtype=np.int32).reshape(B, 2)
        d_off = torch.from_numpy(off[:B].copy()).to(self.device)
        d_hw = torch.from_numpy(hw).to(self.device)
        out = torch.empty((B, dh, dw, 3), dtype=torch.uint8, device=self.device)
        N.check(self.lib.mrx_cv2_resize_u8c3_batch(
            d_src, d_off, d_hw, out, B, dh, dw, N.stream_ptr(stream)),
            "mrx_cv2_resize_u8c3_batch")
        if d_status is not None:
            self.jpeg_check(d_status, jidx)
        if not return_sources:
            return out
        sources = [d_src[int(off[b]):int(off[b]) + int(np.prod(shapes[b]))].view(shapes[b])
                   if b in jidx else images[b] for b in range(B)]
        return out, sources

    def mold_batch_device(self, d_imgs, out_dtype=np.float32, stream=None):
        """resize_image + mold_image for uint8 [B,h,w,3] device images of one size, one launch.
        Returns (molded [B,oh,ow,3], window, scale, padding)."""
        torch = _torch()
        cfg = self.config
        B, h, w = int(d_imgs.shape[0]), int(d_imgs.shape[1]), int(d_imgs.shape[2])
        nh, nw, top, left, oh, ow, window, scale, padding = resize_image_geometry(
            h, w, cfg.IMAGE_MIN_DIM, cfg.IMAGE_MAX_DIM, cfg.IMAGE_MIN_SCALE,
            cfg.IMAGE_RESIZE_MODE)
        out = torch.empty((B, oh, ow, 3), dtype=_torch_dtype(out_dtype), device=self.device)
        mean = [float(v) for v in np.asarray(cfg.MEAN_PIXEL, dtype=np.float64)]
        N.check(self.lib.mrx_mold_image_batch(
            d_imgs, B, h, w, nh, nw, top, left, oh, ow, N.double_array(mean),
            _dtype_code(out_dtype), out, None, N.stream_ptr(stream)),
            "mrx_mold_image_batch")
        return out, window, scale, padding


class StreamingUnmolder:
    """Host-buffer pipeline around UnmoldEngine for a stream of equally-shaped batches:
    the H2D copy of batch k+1 (own stream, double-buffered device inputs) overlaps the D2H
    copy of batch k's masks (PCIe is full duplex); results land in double-buffered pinned
    host memory and are valid after `wait(k)`.

        sm = StreamingUnmolder(engine, geoms)
        for k, (h_det, h_msk) in enumerate(batches):      # pinned [n,R,6] / [n,R,mh,mw,C]
            sm.submit(h_det, h_msk)
            if k: counts, boxes, masks = sm.wait(k - 1)

    packed=True (EXTENSION, not the reference layout): the expand kernel writes bit-packed masks
    (`mrx_mask_expand_packed`) and only those travel back: 8x fewer D2H bytes; the host buffer
    then holds, per image, uint8 [R, H, ceil(W/8)] at `engine.packed_layout()` offsets.

    mask_upload="zero_copy": `mrcnn_mask` is not copied to the device at all -- the class-tile
    gather kernel reads the 1/C of it that is needed straight from the pinned host buffer over
    PCIe (detections are still copied: 2.4 KB per image)."""

    def __init__(self, engine, geoms, packed=False, mask_upload="copy"):
        torch = _torch()
        if mask_upload not in ("copy", "zero_copy"):
            raise ValueError("mask_upload: 'copy' or 'zero_copy'")
        self.eng = engine
        self.packed = bool(packed)
        self.zero_copy = mask_upload == "zero_copy"
        engine.plan(geoms, canvas=False)       # the outputs live here, double-buffered
        n = self.n = engine.layout.n
        dev = engine.device
        det_t, msk_t = _torch_dtype(engine.det_dtype), _torch_dtype(engine.mask_dtype)
        self.d_det = [torch.empty((n, engine.R, 6), dtype=det_t, device=dev) for _ in range(2)]
        self.d_msk = None if self.zero_copy else [
            torch.empty((n, engine.R, engine.mh, engine.mw, engine.C), dtype=msk_t, device=dev)
            for _ in range(2)]
        self.total = engine.packed_layout()[1] if self.packed else int(engine.layout.canvas_off[-1])
        self.d_out = [torch.empty((self.total,), dtype=torch.uint8, device=dev) for _ in range(2)]
        self.h_out = [torch.empty((self.total,), dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.h_counts = [torch.empty((n,), dtype=torch.int32).pin_memory() for _ in range(2)]
        self.h_boxes = [torch.empty((n, engine.R, 4), dtype=torch.int32).pin_memory()
                        for _ in range(2)]
        # three streams: inputs up, kernels, results down -- batch k's download overlaps batch
        # k+1's kernels and batch k+2's upload (PCIe is full duplex)
        self.in_stream = torch.cuda.Stream(device=dev)
        self.out_stream = torch.cuda.Stream(device=dev)
        self.main_stream = torch.cuda.current_stream(dev)
        self.h2d_done = [torch.cuda.Event() for _ in range(2)]
        self.in_free = [torch.cuda.Event() for _ in range(2)]
        self.out_ready = [torch.cuda.Event() for _ in range(2)]
        self.out_free = [torch.cuda.Event() for _ in range(2)]
        self.out_done = {}
        self.k = 0
        msk_bytes = n * engine.R * engine.mh * engine.mw * engine.C * engine.mask_dtype.itemsize
        self.h2d_bytes = self.d_det[0].numel() * self.d_det[0].element_size() + \
            (0 if self.zero_copy else msk_bytes)
        # zero copy: the gather kernel pulls one 32-byte sector per wanted element over PCIe
        self.pcie_read_bytes = n * engine.R * engine.mh * engine.mw * 32 if self.zero_copy else 0
        self.d2h_bytes = self.total + 4 * (n + 4 * n * engine.R)

    def submit(self, h_det, h_msk):
        """Queue one batch (pinned host tensors).  The host buffers of batch k are reused by
        batch k+2: consume `wait(k)`'s result before submitting batch k+2."""
        torch = _torch()
        k, i = self.k, self.k % 2
        eng = self.eng
        if self.zero_copy and not h_msk.is_pinned():
            raise ValueError("zero_copy needs the mask tensor in pinned host memory")
        with torch.cuda.stream(self.in_stream):
            if k >= 2:
                self.in_stream.wait_event(self.in_free[i])     # kernels of batch k-2 read d_*[i]
            self.d_det[i].copy_(h_det, non_blocking=True)
            if not self.zero_copy:
                self.d_msk[i].copy_(h_msk, non_blocking=True)
            self.h2d_done[i].record(self.in_stream)
        ms = self.main_stream
        ms.wait_event(self.h2d_done[i])
        if k >= 2:
            ms.wait_event(self.out_free[i])                    # download of batch k-2 read d_out[i]
        msk = h_msk if self.zero_copy else self.d_msk[i]
        eng.enqueue(self.d_det[i], msk, ms, expand=False)
        if self.packed:
            eng.enqueue_expand_packed(ms, packed_ptr=self.d_out[i].data_ptr())
        else:
            eng.enqueue_expand(ms, canvas_ptr=self.d_out[i].data_ptr())
        self.in_free[i].record(ms)
        # counts / boxes are single-buffered in the engine: copy them (50 KB) before the next
        # batch's prologue overwrites them, on the kernel stream
        with torch.cuda.stream(ms):
            self.h_counts[i].copy_(eng.d_counts[:self.n], non_blocking=True)
            self.h_boxes[i].copy_(eng.d_boxes[:self.n], non_blocking=True)
        self.out_ready[i].record(ms)
        with torch.cuda.stream(self.out_stream):
            self.out_stream.wait_event(self.out_ready[i])
            self.h_out[i].copy_(self.d_out[i], non_blocking=True)
            self.out_free[i].record(self.out_stream)
            ev = torch.cuda.Event()
            ev.record(self.out_stream)
        self.out_done[k] = ev
        self.k += 1
        return k

    def wait(self, k):
        """Block until batch k's results are in pinned host memory; returns
        (counts [n] int32, boxes [n,R,4] int32, output bytes uint8) as torch CPU tensors."""
        self.out_done.pop(k).synchronize()
        i = k % 2
        return self.h_counts[i], self.h_boxes[i], self.h_out[i]
