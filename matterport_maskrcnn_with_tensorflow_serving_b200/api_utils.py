"""Drop-in for the reference's `api.helpers.utils` (imported as `api_utils`,
serve.py:21): same function names, positional arguments, return tuples and
NumPy value semantics, computed by the sm_90a kernels in libmrx.so.

    get_anchors(image_shape)                                         serve.py:105
    unmold_detections(detections, mrcnn_mask, original_image_shape,
                      image_shape, window)                           serve.py:147-154
    load_img(path)                                                   serve.py:86

Plus batched entry points the reference lacks (it is hard-wired to one image per call,
serve.py:48): `unmold_detections_batch`, `unmold_detections_packed_batch`,
`unmold_detections_rle_batch`, `unmold_detections_contours_batch`, `unmold_overlay_batch`,
`unmold_coco_results_batch` (upstream's `build_coco_results` of the unmolded detections),
`unmold_compute_ap_batch` (upstream's `compute_ap` of them against ground truth) and
`unmold_coco_eval_batch` (pycocotools' COCOeval "segm" of them, streamed batch by batch), and
`decode_jpeg_batch` / `decode_png_batch` / `encode_png_batch` / `encode_jpeg_batch` (request
JPEG or PNG bytes in, response PNG or JPEG bytes out, each as OpenCV would decode or write them).

Numerical contract (checked by tests/ against the float64 oracle): N, boxes, class ids and
scores are bit-exact.  The mask resize runs in float32 on exact integer source coordinates;
its pre-threshold samples are within 1e-6 of the reference's float64 values, so a mask pixel
can differ from the reference only where the reference's own value is within 1e-6 of the 0.5
threshold (none on the seeded test data).

Thread safety: these functions may be called from several threads (a threaded web server);
the cached engines are guarded by a lock held from planning a batch until its results are on
the host, so calls are serialised per (device, shape) engine, never interleaved.
"""
from __future__ import annotations

import threading
import weakref
from collections import OrderedDict

import numpy as np

from . import _native as N
from .engine import AnchorGenerator, UnmoldEngine, make_geom
from .model_configs import mconfig as _default_config

_state = {"config": _default_config, "anchors": None, "engines": OrderedDict()}
_state_lock = threading.RLock()
_jpeg_lock = threading.Lock()

# at most this many cached engines (one per device / R / mask shape / dtypes); the least
# recently used one is released (its canvas and input buffers freed) when a new one is needed
MAX_CACHED_ENGINES = 4


def set_config(config):
    """Use another Matterport-style config object (attribute names of mrcnn/config.py)."""
    with _state_lock:
        _state["config"] = config
        _state["anchors"] = None


def get_config():
    return _state["config"]


def release():
    """Free every cached device buffer (engines, anchor memo, pinned result pool)."""
    with _state_lock:
        for eng in _state["engines"].values():
            eng.release()
            eng._inputs = None
        _state["engines"].clear()
        _state["anchors"] = None
        _state.pop("molder", None)
        _pool.clear()


def load_img(path):
    """serve.py:85-86: file -> HxWx3 uint8 RGB ndarray (file IO; stays on the host)."""
    import cv2

    img = cv2.imread(path, cv2.IMREAD_COLOR)
    if img is None:
        raise FileNotFoundError(path)
    return cv2.cvtColor(img, cv2.COLOR_BGR2RGB)


def decode_jpeg_batch(blobs):
    """JPEG files (bytes, bytearray or memoryview) -> one uint8 [H, W, 3] RGB CUDA tensor each,
    equal bit for bit to `load_img` of the same file (cv2.imdecode, BGR -> RGB), decoded on the
    device (csrc/jpeg.cu), sequential and progressive files alike, mixed in one batch.  A file
    the decoder does not accept raises ValueError naming its index
    and the reason before anything is uploaded; corrupt entropy-coded data raises ValueError after
    the decode (libjpeg-turbo would warn and substitute zeros)."""
    from .engine import Molder

    with _jpeg_lock:     # the decoder's buffers are reused; other api_utils calls do not wait
        m = _state.get("molder")
        if m is None or m.config is not get_config():
            m = _state["molder"] = Molder(get_config())
        return m.decode_jpeg_batch(list(blobs))


def decode_png_batch(blobs):
    """PNG files (bytes, bytearray or memoryview) -> one uint8 [H, W, 3] RGB CUDA tensor each,
    equal bit for bit to `load_img` of the same file (cv2.imdecode, BGR -> RGB), decoded on the
    device (csrc/png_decode.cu): every colour type and bit depth, Adam7, EXIF orientation.  A file
    the decoder does not accept raises ValueError naming its index and the reason before anything
    is uploaded; corrupt image data (a CRC, code, distance, Adler-32 or filter error libpng would
    refuse) raises ValueError after the decode."""
    from .engine import Molder

    with _jpeg_lock:     # the decoders share the Molder's buffers
        m = _state.get("molder")
        if m is None or m.config is not get_config():
            m = _state["molder"] = Molder(get_config())
        return m.decode_png_batch(list(blobs))


def encode_png_batch(images):
    """uint8 RGB [H, W, 3] images (CUDA tensors or arrays; sizes may differ) -> one PNG file's
    bytes each, equal byte for byte to `cv2.imencode('.png', img[..., ::-1])[1].tobytes()`,
    encoded on the device (csrc/png.cu).  An image the encoder does not accept raises ValueError
    naming its index before anything runs.  Only the files travel to the host."""
    return _png_encode(images)[0]


def _image_meta(images):
    """(shape, dtype) of each image, CUDA tensor or array, for an encoder's plan."""
    import torch

    meta = []
    for img in images:
        if torch.is_tensor(img):
            meta.append((tuple(img.shape), str(img.dtype).replace("torch.", "")))
        else:
            a = np.asarray(img)
            meta.append((a.shape, a.dtype))
    return meta


def _device_images(images):
    """(device, contiguous uint8 tensors on it): the images an encoder reads in place, on the
    device of the first CUDA tensor among them, else the current one."""
    import torch

    dev = next((im.device for im in images if torch.is_tensor(im) and im.is_cuda),
               torch.device("cuda", torch.cuda.current_device()))
    srcs = []
    for img in images:
        t = img if torch.is_tensor(img) else torch.from_numpy(np.ascontiguousarray(img))
        srcs.append(t.to(dev, non_blocking=True).contiguous())
    return dev, srcs


def _download_files(d_out, offs, d_sizes):
    """The files at offsets offs of d_out, d_sizes[b] bytes each, as one copy to the host."""
    import torch

    sizes = d_sizes.cpu().numpy()
    files = torch.cat([d_out[int(o):int(o) + int(s)] for o, s in zip(offs, sizes)]).cpu()
    host = files.numpy().tobytes()
    ends = np.cumsum(sizes)
    return [host[int(e - s):int(e)] for s, e in zip(sizes, ends)]


def _png_encode(images, stats=False):
    """`encode_png_batch`, plus (with stats) the device's per-image and per-block int64 tables
    (mrx.h MRX_PNG_IMG_* / MRX_PNG_BLK_*) and the plan."""
    import torch

    from . import png

    images = list(images)
    if len(images) == 0:
        return ([], None, None, None) if stats else ([],)
    N.require_cuda()
    plan = png.Plan(_image_meta(images))
    dev, srcs = _device_images(images)
    plan.set_sources([t.data_ptr() for t in srcs])
    lib = N.load()

    def buf(n, dtype):
        return torch.empty(int(n), dtype=dtype, device=dev)

    d_desc = torch.from_numpy(plan.desc).to(dev)
    d_stream, d_sym = buf(plan.stream_bytes, torch.uint8), buf(plan.stream_bytes, torch.int16)
    d_stretch = buf(plan.stretch_words, torch.int32)
    d_tiles = buf(2 * (plan.total_tiles + 1), torch.int64)
    d_blk_pos = buf(plan.blkpos_words, torch.int32)
    d_blk_tab = buf(plan.blocks * png.BLK_TAB_WORDS, torch.int32)
    d_blk_info = buf(plan.blocks * png.BLK_INFO_WORDS, torch.int64)
    d_zbuf = buf(plan.zbuf_words, torch.int32)
    d_img_info = buf(plan.B * png.IMG_INFO_WORDS, torch.int64)
    d_out = buf(plan.out_bytes, torch.uint8)
    d_sizes = buf(plan.B, torch.int64)
    with torch.cuda.device(dev):
        N.check(lib.mrx_png_encode(
            d_desc, plan.B, plan.max_n, plan.max_blocks, plan.max_chunks, plan.total_tiles,
            plan.zbuf_words, d_stream, d_sym, d_stretch, d_tiles, d_blk_pos, d_blk_tab,
            d_blk_info, d_zbuf, d_img_info, d_out, d_sizes, N.stream_ptr()), "mrx_png_encode")
        out = _download_files(d_out, plan.desc[:, png.D_OUT_OFF], d_sizes)
    if not stats:
        return (out,)
    return out, d_img_info.view(plan.B, -1).cpu().numpy(), \
        d_blk_info.view(plan.blocks, -1).cpu().numpy(), plan


def encode_jpeg_batch(images, quality=95, optimize=False):
    """uint8 RGB [H, W, 3] images (CUDA tensors or arrays; sizes may differ) -> one JPEG file's
    bytes each, equal byte for byte to `cv2.imencode('.jpg', img[..., ::-1],
    [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize)])[1].tobytes()`,
    encoded on the device (csrc/jpeg_encode.cu): baseline, 4:2:0, the standard Huffman tables or
    with `optimize` each image's optimal ones.  An image or quality the encoder does not accept
    raises ValueError (naming the image's index) before anything runs.  Only the files travel to
    the host."""
    return _jpeg_encode(images, quality, optimize)[0]


def _jpeg_encode(images, quality=95, optimize=False, stats=False):
    """`encode_jpeg_batch`, plus (with stats) the device's per-image int64 table
    (mrx.h MRX_JPEG_ENC_*), every block's quantised zigzag coefficients (int16 [blocks, 64], the
    plan's D_BLK_OFF rows per image) and the plan."""
    import torch

    from . import jpeg_encode as je

    images = list(images)
    plan = je.EncodePlan(_image_meta(images), quality, optimize)
    if len(images) == 0:
        return ([], None, None, plan) if stats else ([],)
    N.require_cuda()
    dev, srcs = _device_images(images)
    plan.set_sources([t.data_ptr() for t in srcs])
    lib = N.load()

    def buf(n, dtype):
        return torch.empty(int(n), dtype=dtype, device=dev)

    B = plan.B
    d_desc = torch.from_numpy(plan.desc).to(dev)
    d_huff = buf(B * 4 * je.TAB_BYTES, torch.uint8)
    d_codes = buf(B * 4 * 256, torch.int32)
    d_hist = buf(B * 4 * 256, torch.int32)
    d_coef = buf(plan.blocks * 64, torch.int16)
    d_blk_bit = buf(plan.blocks, torch.int32)
    d_tiles = buf(plan.block_tiles + plan.byte_tiles + 2, torch.int64)
    d_words = buf(plan.words, torch.int32)
    d_info = buf(B * je.INFO_WORDS, torch.int64)
    d_out = buf(plan.out_bytes, torch.uint8)
    d_sizes = buf(B, torch.int64)
    with torch.cuda.device(dev):
        N.check(lib.mrx_jpeg_encode(
            d_desc, B, plan.quality, int(plan.optimize), plan.min_side, plan.max_side,
            plan.max_blocks, plan.max_bytes, plan.block_tiles, plan.byte_tiles, plan.words,
            d_huff, d_codes, d_hist, d_coef, d_blk_bit, d_tiles, d_words, d_info, d_out,
            d_sizes, N.stream_ptr()), "mrx_jpeg_encode")
        out = _download_files(d_out, plan.desc[:, je.D_OUT_OFF], d_sizes)
    if not stats:
        return (out,)
    return out, d_info.view(B, -1).cpu().numpy(), d_coef.view(plan.blocks, 64).cpu().numpy(), \
        plan


def get_anchors(image_shape):
    """[A,4] float32 normalised (y1,x1,y2,x2) FPN anchors for a molded image shape;
    memoised by shape like upstream MaskRCNN.get_anchors."""
    with _state_lock:
        if _state["anchors"] is None:
            _state["anchors"] = AnchorGenerator(_state["config"])
        return _state["anchors"].get_anchors(image_shape)


# ----------------------------------------------------------------------------- host results
class _PinnedPool:
    """Pinned host buffers for results handed to the caller as NumPy arrays without an extra
    copy: a buffer goes back to the pool when the last array viewing it is garbage collected
    (pinning 100 MB costs far more than the copy it carries, so buffers are reused)."""

    GRANULE = 1 << 20
    MAX_BYTES = 4 << 30

    def __init__(self):
        self.free = {}
        self.bytes = 0
        self.lock = threading.Lock()

    def clear(self):
        with self.lock:
            self.free.clear()
            self.bytes = 0

    def _give_back(self, size, tensor):
        with self.lock:
            if self.bytes + size <= self.MAX_BYTES:
                self.free.setdefault(size, []).append(tensor)
                self.bytes += size

    def take(self, nbytes):
        """(tensor uint8 [nbytes] pinned, release hook to attach to the final ndarray)."""
        import torch

        size = max(self.GRANULE, (int(nbytes) + self.GRANULE - 1) // self.GRANULE * self.GRANULE)
        with self.lock:
            lst = self.free.get(size)
            t = lst.pop() if lst else None
            if t is not None:
                self.bytes -= size
        if t is None:
            t = torch.empty((size,), dtype=torch.uint8).pin_memory()
        return t, size

    def as_array(self, tensor, size, nbytes):
        """uint8 ndarray [nbytes] viewing `tensor`; the buffer returns to the pool when the
        array (and everything derived from it) is gone."""
        arr = tensor[:nbytes].numpy()
        weakref.finalize(arr.base, self._give_back, size, tensor)
        return arr


_pool = _PinnedPool()


# ----------------------------------------------------------------------------- staging
def _squeeze_inputs(detections, mrcnn_mask):
    detections = np.asarray(detections)
    mrcnn_mask = np.asarray(mrcnn_mask)
    # serve.py:131-136 reshapes to (-1, *cf.OUT_*_SHAPE): accept the leading unit dim
    if detections.ndim == 3 and detections.shape[0] == 1:
        detections = detections[0]
    if mrcnn_mask.ndim == 5 and mrcnn_mask.shape[0] == 1:
        mrcnn_mask = mrcnn_mask[0]
    if detections.ndim != 2 or detections.shape[1] != 6:
        raise ValueError(f"detections must be [R,6], got {detections.shape}")
    if mrcnn_mask.ndim != 4 or mrcnn_mask.shape[0] != detections.shape[0]:
        raise ValueError(f"mrcnn_mask must be [R,mh,mw,C] with R={detections.shape[0]}, "
                         f"got {mrcnn_mask.shape}")
    if detections.dtype not in (np.float32, np.float64):
        detections = detections.astype(np.float64)
    if mrcnn_mask.dtype not in (np.float32, np.float64):
        mrcnn_mask = mrcnn_mask.astype(np.float64)
    return np.ascontiguousarray(detections), np.ascontiguousarray(mrcnn_mask)


def _engine_for(batch, R, mh, mw, Cc, det_dtype, mask_dtype):
    import torch

    key = (torch.cuda.current_device(), R, mh, mw, Cc, np.dtype(det_dtype).str,
           np.dtype(mask_dtype).str)
    with _state_lock:
        engines = _state["engines"]
        eng = engines.get(key)
        if eng is not None and eng.B < batch:
            eng.release()
            eng._inputs = None
            eng = None
        if eng is None:
            while len(engines) >= MAX_CACHED_ENGINES:
                _, old = engines.popitem(last=False)
                old.release()
                old._inputs = None
            eng = UnmoldEngine(max(batch, 1), R, (mh, mw), Cc, det_dtype, mask_dtype)
            eng._inputs = None
        engines[key] = eng
        engines.move_to_end(key)
    return eng


class _Staged:
    """One batch on its engine: inputs uploaded, geometry planned, engine lock HELD until
    `close()` (use as a context manager)."""

    def __init__(self, items, canvas=True):
        import torch

        N.require_cuda()
        dets, masks, geoms = [], [], []
        for det, msk, osh, ish, win in items:
            d, m = _squeeze_inputs(det, msk)
            dets.append(d)
            masks.append(m)
            geoms.append(make_geom(osh, ish, win))
        d0, m0 = dets[0], masks[0]
        for d, m in zip(dets, masks):
            if d.shape != d0.shape or m.shape != m0.shape or d.dtype != d0.dtype or \
                    m.dtype != m0.dtype:
                raise ValueError("all images of a batch must share shapes and dtypes")
        self.n = n = len(items)
        R, (mh, mw, Cc) = d0.shape[0], m0.shape[1:]
        self.eng = eng = _engine_for(n, R, mh, mw, Cc, d0.dtype, m0.dtype)
        eng.lock.acquire()
        try:
            eng.plan(geoms, canvas=canvas)
            # cached device inputs: no np.stack, no per-call device allocation
            if eng._inputs is None:
                from .engine import _torch_dtype
                eng._inputs = (
                    torch.empty((eng.B, R, 6), dtype=_torch_dtype(d0.dtype), device=eng.device),
                    torch.empty((eng.B, R, mh, mw, Cc), dtype=_torch_dtype(m0.dtype),
                                device=eng.device))
            d_det, d_msk = eng._inputs
            for b in range(n):
                # (a read-only ndarray -- a zero-copy view of a received message, wire.py -- is
                # fine here: it is only read)
                d_det[b].copy_(_as_tensor(dets[b]), non_blocking=True)
                d_msk[b].copy_(_as_tensor(masks[b]), non_blocking=True)
            self.d_det, self.d_msk = d_det[:n], d_msk[:n]
        except BaseException:
            eng.lock.release()
            raise

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.eng.lock.release()
        return False

    def meta(self):
        counts, boxes, class_ids, scores = self.eng.fetch_meta()
        return counts, [(boxes[b, :int(counts[b])].copy(), class_ids[b, :int(counts[b])].copy(),
                         scores[b, :int(counts[b])].copy()) for b in range(self.n)]


def _as_tensor(arr):
    import torch
    import warnings

    if arr.flags.writeable:
        return torch.from_numpy(arr)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")     # "non-writable tensors are not supported": read only here
        return torch.from_numpy(arr)


def _download(views):
    """views: contiguous device uint8 tensors.  One pinned buffer per view from the pool, async
    copies, one synchronisation; returns uint8 ndarrays of the views' shapes."""
    import torch

    taken = []
    for v in views:
        nbytes = v.numel()
        if nbytes == 0:
            taken.append(None)
            continue
        t, size = _pool.take(nbytes)
        t[:nbytes].copy_(v.view(-1), non_blocking=True)
        taken.append((t, size, nbytes))
    torch.cuda.current_stream().synchronize()
    return [np.empty(tuple(v.shape), np.uint8) if x is None else
            _pool.as_array(*x).reshape(tuple(v.shape)) for v, x in zip(views, taken)]


# ----------------------------------------------------------------------------- entry points
def unmold_detections_batch(items):
    """items: sequence of (detections, mrcnn_mask, original_image_shape, image_shape,
    window) with equal R / mask shape / dtypes.  Returns a list of
    (boxes, class_ids, scores, masks) as `unmold_detections` returns them per image (see the
    module docstring for the numerical contract)."""
    if len(items) == 0:
        return []
    with _Staged(items) as st:
        eng = st.eng
        eng.enqueue(st.d_det, st.d_msk)
        counts, metas = st.meta()
        arrays = _download([eng.canvas_view(b, counts[b]) for b in range(st.n)])
    # upstream returns np.empty(shape[:2] + (0,)) for no instances
    return [metas[b] + (a.view(np.bool_) if a.shape[2] else np.empty(a.shape),)
            for b, a in enumerate(arrays)]


def unpack_masks(packed, width):
    """Inverse of the packed transport: uint8 [N, H, ceil(W/8)] -> bool [H, W, N] (the array
    `unmold_detections` returns)."""
    if packed.shape[0] == 0:
        return np.empty((packed.shape[1], width, 0))
    return np.unpackbits(packed, axis=-1, count=width).transpose(1, 2, 0).astype(np.bool_)


def unmold_detections_packed_batch(items, direct=True):
    """EXTENSION (not the reference layout): like `unmold_detections_batch` but the masks come
    back bit-packed, uint8 [N, H, ceil(W/8)] with packed[n, y] == np.packbits(masks[y, :, n]) --
    8x less device -> host traffic; `unpack_masks(packed, W)` restores the reference array.

    direct=True: the expand kernel writes the bits itself (`mrx_mask_expand_packed`; the byte
    canvas is never materialised).  direct=False: byte canvas first, then `mrx_pack_masks`
    (also what mask tiles wider than `MRX_MAX_LANE_MASK_W` columns take).  Both give identical
    bytes."""
    if len(items) == 0:
        return []
    with _Staged(items, canvas=not direct) as st:
        st.eng.enqueue_packed(st.d_det, st.d_msk, direct=direct)
        counts, metas = st.meta()
        arrays = _download([st.eng.packed_view(b, counts[b]) for b in range(st.n)])
    return [metas[b] + (a,) for b, a in enumerate(arrays)]


def unmold_detections_rle_batch(items, compressed=False):
    """EXTENSION (not the reference layout): like `unmold_detections_batch` but every mask comes
    back as a COCO run-length encoding -- pycocotools' "uncompressed RLE" dict
    {'size': [H, W], 'counts': uint32 array} (column-major runs starting with zeros) -- computed
    on the device straight from the 28x28 tiles; the [H,W,N] masks are never materialised and
    only the run lengths (a few KB per mask) travel to the host.  Decoding a result gives exactly
    the mask `unmold_detections` returns.  Returns a list of (boxes, class_ids, scores, rles).

    compressed=True: every dict is {'size': [H, W], 'counts': bytes}, pycocotools' compressed RLE,
    byte for byte what `pycocotools.mask.encode(np.asfortranarray(mask))` returns for that mask.
    The strings are made on the device (`mrx_rle_strings`); only they and their offsets travel to
    the host.  `counts.decode("ascii")` makes a dict JSON can hold."""
    if len(items) == 0:
        return []
    with _Staged(items, canvas=False) as st:
        eng = st.eng
        layout = eng.layout
        eng.enqueue(st.d_det, st.d_msk, expand=False)
        if compressed:
            d_str, d_str_off = eng.enqueue_rle_strings()
            counts, metas = st.meta()
            soff = d_str_off.cpu().numpy()
            blob = d_str[:int(soff[-1])].cpu().numpy().tobytes()
            encoding = lambda i: blob[int(soff[i]):int(soff[i + 1])]  # noqa: E731
        else:
            d_runs, off = eng.enqueue_rle()
            counts, metas = st.meta()
            runs = d_runs.cpu().numpy().view(np.uint32)
            encoding = lambda i: runs[int(off[i]) + i:int(off[i + 1]) + i + 1].copy()  # noqa: E731
    rles = [[] for _ in range(st.n)]
    for b, _, i in layout.kept_instances(counts):
        rles[b].append({"size": list(layout.hw(b)), "counts": encoding(i)})
    return [metas[b] + (rles[b],) for b in range(st.n)]


def unmold_coco_results_batch(items, image_ids, category_ids=None):
    """`unmold_detections` followed by upstream's `build_coco_results` (Matterport
    samples/coco/coco.py) in one device pass: a flat list with one dict per kept instance, images
    in order,

        {"image_id": image_ids[b], "category_id": int(category_ids[class_id]),
         "bbox": [x1, y1, x2 - x1, y2 - y1], "score": float(score),
         "segmentation": {"size": [H, W], "counts": bytes}}

    the values upstream builds: `bbox` from the kept boxes as Python ints, `segmentation` the
    compressed RLE of `unmold_detections_rle_batch(items, compressed=True)`.  `category_ids` maps
    class ids to dataset category ids, as upstream's `dataset.get_source_class_id` does; None keeps
    the class id.  items as for `unmold_detections_batch`, one image id per item.  (Upstream takes
    one image's detections and repeats them for every id in its `image_ids`; here each item has its
    own id.)"""
    if len(image_ids) != len(items):
        raise ValueError(f"{len(items)} items but {len(image_ids)} image ids")
    out = []
    for image_id, (rois, class_ids, scores, rles) in zip(
            image_ids, unmold_detections_rle_batch(items, compressed=True)):
        for i in range(rois.shape[0]):
            y1, x1, y2, x2 = (int(v) for v in rois[i])
            cid = int(class_ids[i])
            out.append({"image_id": image_id,
                        "category_id": cid if category_ids is None else int(category_ids[cid]),
                        "bbox": [x1, y1, x2 - x1, y2 - y1],
                        "score": float(scores[i]),
                        "segmentation": rles[i]})
    return out


def unmold_compute_ap_batch(items, gts, iou_thresholds=(0.5,), score_threshold=0.0):
    """`unmold_detections` scored against ground truth without the masks leaving the device:
    for every image b and threshold t, upstream's
    `compute_ap(*gts[b], *unmold_detections(*items[b]), t)` (Matterport `mrcnn.utils`, with
    `score_threshold` passed on to its `compute_matches`).  gts[b] = (gt_boxes [M,4],
    gt_class_ids [M], gt_masks [H,W,M]) in image b's original shape; gt_boxes are `trim_zeros`-ed
    and the masks and class ids cut to the rows left, as upstream does.  The predicted masks are
    bit-packed on the device, the ground truth is packed there too, and the IoUs and matches are
    computed there (`evaluate` has the NumPy drop-ins and states the tie order).  Returns one dict
    per image: `rois`, `class_ids`, `scores` (as `unmold_detections` returns them), `overlaps`
    [N, M] (float32, rows in descending score order; float64 zeros when N or M is 0), and
    `pred_match` [T, N], `gt_match` [T, M] (float64) and `ap` [T] for the T thresholds.

    COCO ground truth: gts[b] = (gt_boxes, gt_class_ids, gt_rles) with gt_rles a list of M RLE
    dicts {'size': [H, W], 'counts': ...} -- compressed strings (`bytes` or `str`, what
    `annToRLE` returns) or uncompressed count lists -- for every image of the batch.  They are
    decoded on the device (`MaskBatch.from_rle`, which raises ValueError for malformed ones), so
    only the strings and runs are uploaded; the results are the same as for the decoded bool
    masks.  gt_rles may also hold COCO polygon or box lists, next to RLE dicts or alone, as a
    COCO instances file gives every non-crowd annotation: they are rasterised on the device as
    pycocotools' annToRLE does (`MaskBatch.from_coco`), with the same results as their RLE.
    gt_boxes may be None: the boxes are then upstream's `extract_bboxes` of the decoded
    masks (y1, x1, y2, x2, exclusive ends, zeros for an empty mask), read from the device with
    one synchronisation, `trim_zeros`-ed and applied as above; that image's dict also has them
    as `gt_rois` (int32 [M, 4])."""
    from . import evaluate

    if len(gts) != len(items):
        raise ValueError(f"{len(items)} items but {len(gts)} ground-truth tuples")
    if len(items) == 0:
        return []
    thresholds = list(iou_thresholds)
    rle = [isinstance(g[2], (list, tuple)) and all(isinstance(r, (dict, list)) for r in g[2])
           for g in gts]
    if any(rle) and not all(rle):
        raise ValueError("ground truth must be bool mask arrays for every image or RLE lists for "
                         "every image")
    rle = all(rle)
    polygons = rle and any(isinstance(r, list) for g in gts for r in g[2])
    gt_cls, gt_masks = [], []
    for boxes, cls, masks in gts:
        if rle and boxes is None:
            gt_cls.append(np.asarray(cls))
            gt_masks.append(list(masks))
            continue
        m = evaluate.trim_zeros(np.asarray(boxes)).shape[0]
        gt_cls.append(np.asarray(cls)[:m])
        gt_masks.append(list(masks)[:m] if rle else np.asarray(masks)[..., :m])
    gt_rois = {}
    with _Staged(items, canvas=False) as st:
        eng = st.eng
        eng.enqueue_packed(st.d_det, st.d_msk)
        if rle:
            gt = (eng.ground_truth_coco if polygons else eng.ground_truth_rle)(gt_cls, gt_masks)
            keep = gt.counts.copy()
            for b, g in enumerate(gts):
                if g[0] is None:
                    gt_rois[b] = gt.extents[b, :keep[b]].copy()
                    keep[b] = evaluate.trim_zeros(gt_rois[b]).shape[0]
            if gt_rois:
                gt.set_counts(keep)
        else:
            gt = eng.ground_truth(gt_cls, gt_masks)
        d_ov = eng.enqueue_overlaps(gt)
        d_order, d_pm, d_gm = eng.enqueue_matches(gt, thresholds, score_threshold)
        counts, metas = st.meta()
        ov, order, pm, gm = (t.cpu().numpy() for t in (d_ov, d_order, d_pm, d_gm))
    out = []
    for b, (rois, class_ids, scores) in enumerate(metas):
        n, m = int(counts[b]), int(gt.counts[b])
        pred_match = pm[:, b, :n].astype(np.float64)
        gt_match = gm[:, b, :m].astype(np.float64)
        out.append({
            "rois": rois, "class_ids": class_ids, "scores": scores,
            "overlaps": ov[b, :n, :m][order[b, :n]] if n and m else np.zeros((n, m)),
            "pred_match": pred_match, "gt_match": gt_match,
            "ap": np.array([evaluate.ap_from_matches(pred_match[t], gt_match[t])[0]
                            for t in range(len(thresholds))]),
        })
        if b in gt_rois:
            out[-1]["gt_rois"] = gt_rois[b]
    return out


def unmold_coco_eval_batch(items, image_ids, gt_anns, evaluator, category_ids=None):
    """`unmold_detections` scored as pycocotools' COCOeval scores segm, bbox or boundary results,
    or as lvis-api's LVISEval scores segm or bbox results, without the masks leaving the device:
    adds the batch to `evaluator` (an `evaluate.COCOevalSegm`, `evaluate.COCOevalBbox`,
    `evaluate.COCOevalBoundary`, `evaluate.LVISEvalSegm` or `evaluate.LVISEvalBbox`), whose
    `accumulate()` and `summarize()` give COCO mask, box or Boundary AP, or LVIS mask or box AP,
    once every batch is in.  items as for `unmold_detections_batch`; image_ids, one per item;
    gt_anns[b], image b's annotation dicts; category_ids as for `unmold_coco_results_batch`.
    Equivalent to `evaluator.add_results(unmold_coco_results_batch(items, image_ids,
    category_ids), gt_anns, image_ids)`, but the predicted masks go straight to packed planes and
    are never encoded, and bbox evaluation expands no mask at all.

    `evaluator` may also be a list of evaluators, e.g. `[COCOevalSegm(), COCOevalBbox(),
    COCOevalBoundary()]` for mask AP, box AP and Boundary AP from one unmold, or
    `[COCOevalSegm(), LVISEvalSegm(categories, images)]` for COCO and LVIS mask AP on the same
    annotations: the items are staged and the prepare step runs once, the packed expand once when
    a segm, boundary or LVIS segm evaluator is among them, and each evaluator gets the records
    its own `add_batch` would give it.  Every evaluator checks the batch before anything runs."""
    evaluators = list(evaluator) if isinstance(evaluator, (list, tuple)) else [evaluator]
    if len({id(e) for e in evaluators}) != len(evaluators):
        raise ValueError("the same evaluator is given twice")
    tables = [e._batch_tables(items, image_ids, gt_anns) for e in evaluators]
    if len(items) == 0:
        return
    with _Staged(items, canvas=False) as st:
        eng = st.eng
        if any(e._needs_masks for e in evaluators):
            eng.enqueue_packed(st.d_det, st.d_msk)
        else:
            eng.enqueue(st.d_det, st.d_msk, expand=False)
        st.meta()                          # raises for bad class ids or boxes
        records = []
        for e, t in zip(evaluators, tables):
            status = e._batch_status(image_ids, t[0])
            gt, t = e._ground_truth(eng.lib, eng.device, eng.layout.geom, t)
            res = e._ious(eng.lib, eng.predictions(gt), gt, t, e._class_map(eng.C, category_ids),
                          status)
            records.append((res, t, status))
    for e, (res, t, status) in zip(evaluators, records):
        e._record(image_ids, res, *t[:3], status)


def unmold_detections_contours_batch(items):
    """EXTENSION: like `unmold_detections_batch` but every instance comes back as the contour
    polygons `visualize.display_instances` draws for it -- a list of float64 [V, 2] (x, y) arrays
    equal to `np.fliplr(v) - 1` of `skimage.measure.find_contours(padded_mask, 0.5)` -- traced on
    the device from the packed masks; only the vertices travel to the host.  Masks with tiles up
    to `MRX_MAX_LANE_MASK_W` columns are expanded straight into bits (`mrx_mask_expand_packed`),
    wider ones through the byte canvas and `mrx_pack_masks`.  Returns a list of (boxes,
    class_ids, scores, contours)."""
    if len(items) == 0:
        return []
    with _Staged(items, canvas=False) as st:
        st.eng.enqueue_packed(st.d_det, st.d_msk)
        counts, metas = st.meta()
        contours = st.eng.enqueue_contours()
    return [metas[b] + (contours[b],) for b in range(st.n)]


def _check_annotate(annotate, class_names):
    if annotate and class_names is None:
        raise ValueError("annotate=True needs class_names for the captions")


def unmold_overlay_batch(items, images, colors=None, alpha=0.5, annotate=False, class_names=None):
    """`unmold_detections` followed by the mask overlay of `visualize.display_instances`
    (serve.py:147-169) without moving the masks to the host: the [H,W,N] canvases stay on
    the device, only boxes, class ids, scores and the blended uint8 images come back.

    items as for `unmold_detections_batch`; images: the original uint8 HxWx3 images;
    colors: RGB triples (shared list, or one list per image; default: `random_colors(R)`).
    annotate=True also draws each instance's box, contour outlines and caption
    "<class_names[class_id]> <score:.3f>" as OpenCV draws them (`visualize.composite_batch`).
    Returns a list of (boxes, class_ids, scores, overlay_uint8)."""
    from . import visualize

    _check_annotate(annotate, class_names)
    if len(items) == 0:
        return []
    with _Staged(items) as st:
        eng = st.eng
        eng.enqueue(st.d_det, st.d_msk)
        if colors is None:
            colors = visualize.random_colors(eng.R)
        overlays = visualize.composite_batch(eng, images, colors, alpha, annotate=annotate,
                                             class_names=class_names)
        counts, metas = st.meta()
        host = [o.cpu().numpy() for o in overlays]
    return [metas[b] + (host[b],) for b in range(st.n)]


def _check_file_format(image_format, quality):
    """Refuse a response format other than "png" or "jpeg", or a JPEG quality cv2 refuses."""
    if image_format not in ("png", "jpeg"):
        raise ValueError(f"image_format {image_format!r} (expected 'png' or 'jpeg')")
    if image_format == "jpeg":
        from .jpeg_encode import check_quality

        check_quality(quality)


def _unmold_overlay_file_batch(items, images, colors=None, alpha=0.5, image_format="png",
                               quality=95, annotate=False, class_names=None):
    """`unmold_overlay_batch` that stops at the device overlays and encodes them there: returns
    (boxes, class_ids, scores, file_bytes) per image, the file being what
    `cv2.imencode('.png', overlay[..., ::-1])` gives for the overlay `unmold_overlay_batch`
    returns (with the same `annotate` and `class_names`), or with image_format "jpeg"
    `cv2.imencode('.jpg', ...)` at `quality`.  Only the file bytes leave the device."""
    from . import visualize

    _check_file_format(image_format, quality)
    _check_annotate(annotate, class_names)
    if len(items) == 0:
        return []
    with _Staged(items) as st:
        eng = st.eng
        eng.enqueue(st.d_det, st.d_msk)
        if colors is None:
            colors = visualize.random_colors(eng.R)
        overlays = visualize.composite_batch(eng, images, colors, alpha, annotate=annotate,
                                             class_names=class_names)
        counts, metas = st.meta()
        if image_format == "jpeg":
            files = encode_jpeg_batch(overlays, quality)
        else:
            files = encode_png_batch(overlays)
    return [metas[b] + (files[b],) for b in range(st.n)]


def unmold_detections(detections, mrcnn_mask, original_image_shape, image_shape, window):
    """Reformat one image's detections from the molded image back to the original image.

    detections: [R, (y1, x1, y2, x2, class_id, score)] normalised coordinates
    mrcnn_mask: [R, mh, mw, num_classes]
    original_image_shape: (H, W, 3) before resizing     image_shape: molded shape
    window: (y1, x1, y2, x2) pixel box of the real image inside the molded image

    Returns boxes [N,4] int32 pixels, class_ids [N] int32, scores [N], masks [H,W,N] bool.
    Boxes, class ids and scores equal the reference's bit for bit; a mask pixel can differ
    only where the reference's float64 resized value is within 1e-6 of the 0.5 threshold.
    """
    return unmold_detections_batch(
        [(detections, mrcnn_mask, original_image_shape, image_shape, window)])[0]
