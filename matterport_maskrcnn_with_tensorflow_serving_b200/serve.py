"""Request/response surface of the reference's serve.py, kept signature for signature:

    preprocess_input(img, img_size=640) -> (molded_image, image_meta, anchors, window)   serve.py:83-107
    grpc_inference(img) -> (mrcnn_detection, mrcnn_mask, molded_image, window)            serve.py:110-138
    do_inference(img) -> save_path                                                        serve.py:141-173

plus the batched surface the reference lacks (it is hard-wired to one image per request,
serve.py:48,53,63,74): `preprocess_input_batch`, `grpc_inference_batch`, `do_inference_batch`,
`do_inference_unmolded` for callers that want the (rois, class_ids, scores, masks) tuple
of serve.py:147 instead of the picture, and `do_inference_coco_batch` for callers that want COCO
result dicts (compressed RLE masks) to answer with JSON.

The TensorFlow-Serving RPC itself (serve.py:26-80) is out of scope and is injected:
`set_predict_fn(fn)` installs `fn(molded_image_f32, image_meta_f32, anchors_f32) ->
(mrcnn_detection, mrcnn_mask)` -- float lists / arrays as `float_val` gives them, or the
`TensorProto` messages themselves (or their bytes), which are then decoded from the wire format
without a Python float per element (`wire.py`); without one `grpc_inference` raises.

`do_inference` ends like the reference (serve.py:156-173): the masks are blended into the
image and the picture is written to `media/mask-<uuid>.png`, whose path is returned.  The
blend runs on the device canvas the unmold kernels just wrote (`mrx_composite_masks`): the
105 MB of masks per 1024x1024x100 image never travel to the host, and neither do the blended
pixels: the PNG file is encoded on the device, byte for byte what `cv2.imwrite` writes
(`api_utils.encode_png_batch`), and only its bytes are downloaded.  `image_format="jpeg"` writes
`media/mask-<uuid>.jpg` instead, the bytes `cv2.imencode('.jpg')` gives at `quality`
(`api_utils.encode_jpeg_batch`), several times smaller than the PNG.  Boxes, captions and
contour polygons are matplotlib artists in the reference; by default they are not drawn.
`annotate=True` draws them on the device as OpenCV draws them (DESIGN.md 3.25), the captions
naming the classes `["BG", *cf.DAMAGE_CLASSES]` as serve.py:165 does; matplotlib's own styling
stays out of scope (DESIGN.md 7).

Wherever an image is accepted, a JPEG or PNG file's bytes (bytes, bytearray or memoryview) are
accepted too, told apart by their signature (`imagefile`): they are decoded on the device
(`api_utils.decode_jpeg_batch`, `api_utils.decode_png_batch`, bit for bit as `load_img`), so the
decoded pixels never reach the host.  A `str` path still goes through `load_img`.
"""
from __future__ import annotations

import os
import threading
import uuid

import numpy as np

from . import api_utils
from . import configs as cf
from . import imagefile, wire
from .engine import Molder

_predict_fn = None
_molder = None
_molder_lock = threading.Lock()


def set_predict_fn(fn):
    global _predict_fn
    _predict_fn = fn


def compose_image_meta(image_id, original_image_shape, image_shape, window, scale,
                       active_class_ids):
    """serve.py:100-103 (upstream model.compose_image_meta): host-side list packing."""
    return np.array(
        [image_id] + list(original_image_shape) + list(image_shape) + list(window) +
        [scale] + list(active_class_ids))


def _get_molder():
    global _molder
    mcf = api_utils.get_config()
    if _molder is None or _molder.config is not mcf:
        _molder = Molder(mcf)
    return _molder


def _is_file(img):
    return isinstance(img, (bytes, bytearray, memoryview))


def _check_image(img, index=0):
    """An image argument: a path (loaded by `load_img`), JPEG or PNG bytes (kept for the device
    decoders; anything else raises ValueError) or an HxWx3 uint8 array."""
    if isinstance(img, str):
        img = api_utils.load_img(img)
    if _is_file(img):
        imagefile.kind(img, index)
        return img
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise TypeError("preprocess_input expects an HxWx3 uint8 image")
    return img


def _image_shape(img):
    """(H, W, 3) of a checked image argument; for a file from its headers alone."""
    if _is_file(img):
        return imagefile.shape(img)
    return tuple(img.shape)


def preprocess_input(img, img_size=640, molded_dtype=np.float64):
    """serve.py:83-107.  molded_dtype float64 reproduces the reference's return value
    (uint8 -> float32 -> minus float64 MEAN_PIXEL); float32 returns exactly what
    serve.py:117 sends on the wire (`molded_image.astype(np.float32)`)."""
    import torch

    mcf = api_utils.get_config()
    img = _check_image(img)
    with _molder_lock:
        molder = _get_molder()
        if _is_file(img):
            d_img, = molder.decode_files([img])
        else:
            d_img = torch.from_numpy(np.ascontiguousarray(img)).to(molder.device)
        if img_size is not None:
            d_img = molder.cv2_resize_device(d_img, (img_size, img_size))
        img_shape = tuple(d_img.shape)
        d_molded, _, window, scale, _padding = molder.mold_device(d_img, out_dtype=molded_dtype)
        molded_image = d_molded.cpu().numpy()
    image_meta = compose_image_meta(
        0, img_shape, molded_image.shape, window, scale,
        np.zeros([mcf.NUM_CLASSES], dtype=np.int32))
    anchors = api_utils.get_anchors(molded_image.shape)
    return molded_image, image_meta, anchors, window


def preprocess_input_batch(imgs, img_size=640, molded_dtype=np.float32):
    """`preprocess_input` for a list of images with one `cv2.resize` launch and one
    `resize_image + mold_image` launch for the whole batch, anchors from the memo.

    With `img_size` given (the reference always passes cf.IMAGE_SIZE, serve.py:114) the inputs
    may have any sizes.  With `img_size=None` they must share one size.  Returns
    (molded_images [B,H,W,3], image_metas [B,M], anchors [A,4] (shared), windows: list of
    4-tuples) -- row b equals `preprocess_input(imgs[b], img_size, molded_dtype)`.
    Default dtype float32: what serve.py:117 puts on the wire."""
    imgs = [_check_image(im, i) for i, im in enumerate(imgs)]
    return _preprocess_batch(imgs, img_size, molded_dtype)[:4]


def _preprocess_batch(imgs, img_size, molded_dtype):
    """`preprocess_input_batch` of checked images, plus each image's pixels for the overlay: the
    array itself, or for file bytes its decoded slot of the buffer the resize read (uint8
    [H, W, 3] on the device, consumed in place)."""
    import torch

    mcf = api_utils.get_config()
    if len(imgs) == 0:
        raise ValueError("empty batch")
    with _molder_lock:
        molder = _get_molder()
        if img_size is not None:
            d_imgs, sources = molder.cv2_resize_batch_device(imgs, (img_size, img_size),
                                                             return_sources=True)
            status = None
        else:
            shapes = [_image_shape(im) for im in imgs]
            if any(sh != shapes[0] for sh in shapes):
                raise ValueError("img_size=None needs equally sized images")
            if not any(_is_file(im) for im in imgs):
                d_imgs = torch.from_numpy(np.stack(imgs)).to(molder.device)
                sources, status = list(imgs), None
            else:
                # one contiguous [B, H, W, 3] buffer: arrays staged, files decoded in place
                d_src, off, _, status, fidx = molder.stage_images(imgs, align=1)
                d_imgs = d_src[:int(off[-1])].view(len(imgs), *shapes[0])
                sources = [d_imgs[b] if b in fidx else imgs[b] for b in range(len(imgs))]
        img_shape = tuple(d_imgs.shape[1:])
        d_molded, window, scale, _padding = molder.mold_batch_device(d_imgs, out_dtype=molded_dtype)
        if status is not None:
            molder.files_check(*status)
        molded = d_molded.cpu().numpy()
    meta = compose_image_meta(0, img_shape, molded.shape[1:], window, scale,
                              np.zeros([mcf.NUM_CLASSES], dtype=np.int32))
    metas = np.stack([meta] * len(imgs))
    anchors = api_utils.get_anchors(molded.shape[1:])
    return molded, metas, anchors, [window] * len(imgs), sources


def _is_tensor_proto(x):
    return isinstance(x, (bytes, bytearray, memoryview)) or hasattr(x, "SerializeToString")


def _decode_outputs(mrcnn_detection, mrcnn_mask):
    if _is_tensor_proto(mrcnn_detection) and _is_tensor_proto(mrcnn_mask):
        # result.outputs[...] handed over as TensorProto messages (or their bytes): take the
        # values from the wire instead of through per-element Python floats (wire.py)
        return wire.decode_predict_outputs(
            mrcnn_detection, mrcnn_mask, cf.OUT_DETECTION_SHAPE, cf.OUT_MASK_SHAPE)
    # serve.py:131-136: float_val lists become float64 arrays with a leading -1 dim
    mrcnn_detection = np.array(mrcnn_detection).reshape((-1, *cf.OUT_DETECTION_SHAPE))
    mrcnn_mask = np.array(mrcnn_mask).reshape((-1, *cf.OUT_MASK_SHAPE))
    return mrcnn_detection, mrcnn_mask


def grpc_inference(img):
    """serve.py:110-138 with the RPC injected (see module docstring)."""
    if _predict_fn is None:
        raise RuntimeError("no TensorFlow-Serving client installed: call set_predict_fn()")
    molded_image, image_meta, anchors, window = preprocess_input(img, cf.IMAGE_SIZE)
    mrcnn_detection, mrcnn_mask = _predict_fn(
        molded_image.astype(np.float32), image_meta.astype(np.float32),
        anchors.astype(np.float32))
    mrcnn_detection, mrcnn_mask = _decode_outputs(mrcnn_detection, mrcnn_mask)
    return mrcnn_detection, mrcnn_mask, molded_image, window


def grpc_inference_batch(imgs):
    """`grpc_inference` for a list of images: batched pre-processing, then one RPC per image
    (the served model's signature is batch 1, serve.py:48).  Returns a list of
    (mrcnn_detection, mrcnn_mask, molded_image_shape, window)."""
    return _grpc_inference_batch([_check_image(im, i) for i, im in enumerate(imgs)])[0]


def _grpc_inference_batch(imgs):
    """`grpc_inference_batch` of checked images, plus each image's pixels (`_preprocess_batch`)."""
    if _predict_fn is None:
        raise RuntimeError("no TensorFlow-Serving client installed: call set_predict_fn()")
    molded, metas, anchors, windows, sources = _preprocess_batch(imgs, cf.IMAGE_SIZE, np.float32)
    anchors32 = anchors.astype(np.float32)
    out = []
    for b in range(len(imgs)):
        det, msk = _predict_fn(molded[b], metas[b].astype(np.float32), anchors32)
        det, msk = _decode_outputs(det, msk)
        out.append((det, msk, molded[b].shape, windows[b]))
    return out, sources


def do_inference_unmolded(img):
    """serve.py:141-154 without the picture: (final_rois, final_class_ids, final_scores,
    final_masks) exactly as `api_utils.unmold_detections` returns them."""
    img = _check_image(img)
    mrcnn_detection, mrcnn_mask, molded_image, window = grpc_inference(img)
    return api_utils.unmold_detections(
        mrcnn_detection, mrcnn_mask, _image_shape(img), molded_image.shape, window)


def _save_file(data, ext, media_dir=None):
    """serve.py:156-158,168: media/mask-<uuid4>.<ext>, the file's bytes encoded on the device
    (what cv2.imwrite of the overlay writes)."""
    media_dir = media_dir if media_dir is not None else getattr(cf, "MEDIA_DIR", "media")
    os.makedirs(media_dir, exist_ok=True)
    save_path = os.path.join(media_dir, "mask-{}.{}".format(str(uuid.uuid4()), ext))
    try:
        with open(save_path, "wb") as f:
            f.write(data)
    except OSError as e:
        raise IOError(f"could not write {save_path}") from e
    return save_path


def do_inference(img, colors=None, media_dir=None, image_format="png", quality=95,
                 annotate=False):
    """serve.py:141-173: inference, unmold, mask overlay, PNG -> `save_path`.  The masks stay
    on the device between the unmold and the overlay (`api_utils.unmold_overlay_batch`).
    image_format "jpeg" writes `media/mask-<uuid>.jpg` instead, the bytes of
    `cv2.imencode('.jpg')` of the overlay at `quality`, encoded on the device.  annotate=True
    also draws the boxes, contour outlines and captions (module docstring)."""
    return do_inference_batch([img], colors=colors, media_dir=media_dir,
                              image_format=image_format, quality=quality, annotate=annotate)[0]


def do_inference_batch(imgs, colors=None, media_dir=None, image_format="png", quality=95,
                       annotate=False):
    """`do_inference` for a list of images: batched pre-processing, one RPC per image, ONE
    batched unmold + overlay on the device, one PNG (or JPEG) per image.  Returns the list of
    paths."""
    api_utils._check_file_format(image_format, quality)
    imgs = [_check_image(im, i) for i, im in enumerate(imgs)]
    if len(imgs) == 0:
        return []
    res, sources = _grpc_inference_batch(imgs)
    items = [(det, msk, tuple(src.shape), mshape, window)
             for (det, msk, mshape, window), src in zip(res, sources)]
    outs = api_utils._unmold_overlay_file_batch(
        items, sources, colors=colors, image_format=image_format, quality=quality,
        annotate=annotate, class_names=["BG", *cf.DAMAGE_CLASSES] if annotate else None)
    ext = "jpg" if image_format == "jpeg" else "png"
    paths = []
    for _boxes, _cls, _scores, data in outs:
        paths.append(_save_file(data, ext, media_dir))
        print(">>> Save image: {}".format(paths[-1]))
    print(">>> Complete!")
    return paths


def do_inference_coco_batch(imgs, image_ids, category_ids=None):
    """The answer of a JSON endpoint instead of a PNG: batched pre-processing, one RPC per image
    (`grpc_inference_batch`), then `api_utils.unmold_coco_results_batch` -- one COCO result dict
    per detected instance, its mask as a compressed RLE made on the device.  image_ids: one per
    image; category_ids: class id -> dataset category id (None: the class id itself).  Decode each
    `segmentation["counts"]` with `.decode("ascii")` before `json.dumps`."""
    imgs = [_check_image(im, i) for i, im in enumerate(imgs)]
    if len(image_ids) != len(imgs):
        raise ValueError(f"{len(imgs)} images but {len(image_ids)} image ids")
    if len(imgs) == 0:
        return []
    res, sources = _grpc_inference_batch(imgs)
    items = [(det, msk, tuple(src.shape), mshape, window)
             for (det, msk, mshape, window), src in zip(res, sources)]
    return api_utils.unmold_coco_results_batch(items, image_ids, category_ids)
