"""GPU test of the package's stream rule (engine.py's module docstring): with a side stream `s`
passed as the `stream` argument of the pipeline launches while the default stream is current, or
made current by `with torch.cuda.stream(s):` for everything else, every libmrx launch of every
family goes to `s`, and every output equals, byte for byte, the same calls on the default
stream."""
import contextlib
import ctypes as C
import random
import re

import cv2
import numpy as np
import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate, synth, visualize
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import (AnchorGenerator, BatchLayout,
                                                                     MaskBatch, Molder,
                                                                     UnmoldEngine, make_geom)

from helpers import item_of

pytestmark = pytest.mark.gpu

NAMES = ["BG", "dent", "scratch", "crack", "glass"]
SHAPES = [(96, 128), (80, 72)]
R = 8

# one launch of each family: what the side-stream run must reach
FAMILIES = {"mrx_unmold_prepare", "mrx_mask_expand", "mrx_mask_expand_packed", "mrx_pack_masks",
            "mrx_rle_count", "mrx_rle_write", "mrx_rle_strings", "mrx_contours_count",
            "mrx_contours_write", "mrx_annotate_draw", "mrx_annotate_resolve", "mrx_mask_extents",
            "mrx_mask_overlaps", "mrx_mask_matches", "mrx_rle_decode", "mrx_poly_decode",
            "mrx_mask_boundary", "mrx_coco_ranks", "mrx_coco_ious", "mrx_coco_box_ious",
            "mrx_coco_boundary_ious", "mrx_coco_match", "mrx_coco_match_f64area",
            "mrx_jpeg_coefficients", "mrx_jpeg_pixels", "mrx_png_decode",
            "mrx_cv2_resize_u8c3_batch", "mrx_mold_image_batch", "mrx_anchors",
            "mrx_composite_masks", "mrx_png_encode", "mrx_jpeg_encode"}


def _stream_functions():
    """Every mrx_* whose prototype in include/mrx.h ends in `void *stream`."""
    with open(N.HEADER_PATH) as f:
        text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)
    return {fn for fn, params in re.findall(r"\b(mrx_\w+)\s*\(([^;{}]*)\)\s*;", text)
            if re.search(r"\bvoid\s*\*\s*stream\s*$", params)}


class _Recorder:
    """libmrx with every launch that takes a stream recording (name, handle) before it runs."""

    def __init__(self, lib, names):
        self._lib, self._names, self.calls = lib, names, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in self._names:
            return fn

        def launch(*args):
            h = args[-1]
            self.calls.append((name, h.value if isinstance(h, C.c_void_p) else h))
            return fn(*args)

        return launch


@pytest.fixture
def recorder(cuda_device, monkeypatch):
    api_utils.release()                  # no cached engine or molder holds the real library
    names = _stream_functions()
    assert FAMILIES <= names
    rec = _Recorder(N.load(), names)
    monkeypatch.setattr(N, "_lib", rec)
    yield rec
    api_utils.release()


def _rle(m):
    """Uncompressed COCO RLE of a bool [H, W] mask."""
    f = np.asarray(m, bool).ravel(order="F")
    ends = np.concatenate([np.flatnonzero(f[1:] != f[:-1]) + 1, [f.size]])
    runs = np.diff(np.concatenate([[0], ends]))
    if f[0]:
        runs = np.concatenate([[0], runs])
    return {"size": list(m.shape), "counts": [int(v) for v in runs]}


def _inputs():
    """Seeded model outputs, images, and ground truth (masks, boxes, polygons) of SHAPES."""
    rng = np.random.default_rng(2024)
    ims = [synth.make_image(rng, hw, 5, num_classes=len(NAMES), max_instances=R) for hw in SHAPES]
    images = [synth.synth_rgb_image(rng, H, W) for H, W in SHAPES]
    cls, masks, anns, polys = [], [], [], []
    for H, W in SHAPES:
        c = rng.integers(1, len(NAMES), size=3).astype(np.int32)
        m = np.zeros((H, W, 3), bool)
        a, p = [], []
        for k in range(3):
            y1, x1 = int(rng.integers(0, H // 2)), int(rng.integers(0, W // 2))
            y2, x2 = y1 + int(rng.integers(8, H // 2)), x1 + int(rng.integers(8, W // 2))
            m[y1:y2, x1:x2, k] = True
            a.append({"category_id": int(c[k]), "segmentation": _rle(m[:, :, k]), "iscrowd": 0,
                      "area": float((y2 - y1) * (x2 - x1)), "bbox": [x1, y1, x2 - x1, y2 - y1],
                      "id": k + 1})
            p.append([[x1, y1, x2, y1 + 3.5, x2 - 2.25, y2, x1 + 1, y2 - 1]])
        cls.append(c)
        masks.append(m)
        anns.append(a)
        polys.append(p)
    return ims, images, cls, masks, anns, polys


def _planes(d_packed, layout, counts):
    """The written planes of a packed output: image b's first counts[b] planes (the rest of each
    slot is never written)."""
    host = d_packed.cpu().numpy()
    return [host[slice(*layout.packed_span(b, k))] for b, k in enumerate(counts)]


def _workload(s):
    """One representative of every family: the pipeline launches given `s` (None: the default
    stream) while the default stream is current, then everything else with `s` made current.
    Returns every output the calls define, on the host (bytes past the kept instances are left
    unwritten by the kernels)."""
    import torch

    ims, images, gt_cls, gt_masks, anns, polys = _inputs()
    geoms = [make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims]
    out = {}
    eng = UnmoldEngine(len(ims), R, (28, 28), len(NAMES))
    d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
    eng.plan(geoms)
    assert torch.cuda.current_stream() == torch.cuda.default_stream()
    eng.enqueue(d_det, d_msk, s)
    d_packed, _ = eng.enqueue_packed(d_det, d_msk, s)
    with torch.cuda.stream(s):
        counts = eng.d_counts[:len(ims)].cpu().numpy()
        out["counts"] = counts
        out["enqueue_packed"] = _planes(d_packed, eng.layout, counts)
    d_packed, _ = eng.enqueue_expand_packed(s)
    with torch.cuda.stream(s):      # the rest on `s` made current
        out["enqueue_expand_packed"] = _planes(d_packed, eng.layout, counts)
        canvas = eng.d_canvas.cpu().numpy()
        out["canvas"] = [canvas[slice(*eng.layout.canvas_span(b, k))]
                         for b, k in enumerate(counts)]

        colors = visualize.random_colors(R, rng=random.Random(5))
        out["pack_masks"] = _planes(eng.pack_masks()[0], eng.layout, counts)
        d_str, d_str_off = eng.enqueue_rle_strings()
        str_off = d_str_off.cpu().numpy()
        out["rle_strings"] = (d_str[:int(str_off[-1])].cpu().numpy(), str_off)
        out["contours"] = eng.enqueue_contours()
        offs = np.cumsum([0] + [H * W * 3 for H, W in SHAPES])
        d_img = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).cuda()
        rgb8 = np.stack([visualize.color_table(colors, R)] * len(ims))
        eng.annotate(d_img, torch.from_numpy(offs[:-1]).cuda(), rgb8,
                     (np.zeros((0, 6), np.int64), np.zeros(0, np.uint8)))
        out["annotate"] = d_img.cpu().numpy()

        gt = eng.ground_truth_rle(gt_cls, [[a["segmentation"] for a in x] for x in anns])
        ov = eng.enqueue_overlaps(gt).cpu().numpy()
        order, pm, gm = (t.cpu().numpy() for t in eng.enqueue_matches(gt, [0.5, 0.75]))
        out["overlaps"] = [ov[b, :k, :gt.counts[b]] for b, k in enumerate(counts)]
        out["matches"] = [(order[b, :k], pm[:, b, :k], gm[:, b, :gt.counts[b]])
                          for b, k in enumerate(counts)]
        mb = MaskBatch.from_coco(eng.lib, eng.device, geoms, gt_cls, polys)
        bp = mb.boundary_planes()
        mb_layout = BatchLayout(mb.geom, mb.R, limits=False)
        out["from_coco"] = (_planes(mb.planes.d_packed, mb_layout, mb.counts), mb.extents)
        out["boundary_planes"] = (_planes(bp.d_packed, mb_layout, mb.counts),
                                  bp.d_areas.cpu().numpy())

        items = [item_of(im, np.float32) for im in ims]
        for ev in (evaluate.COCOevalSegm(), evaluate.COCOevalBbox(), evaluate.COCOevalBoundary()):
            ev.add_batch(items, [11, 12], anns)
            out[type(ev).__name__] = (ev._dets, ev._gts)

        m = Molder(api_utils.get_config())
        jpg = cv2.imencode(".jpg", images[0][:, :, ::-1])[1].tobytes()
        png = cv2.imencode(".png", images[1][:, :, ::-1])[1].tobytes()
        out["decode_files"] = [t.cpu().numpy() for t in m.decode_files([jpg, png])]
        d_small = m.cv2_resize_batch_device([images[0], jpg, png], (64, 64))
        out["cv2_resize_batch"] = d_small.cpu().numpy()
        molded, window, scale, padding = m.mold_batch_device(d_small)
        out["mold_batch"] = (molded.cpu().numpy(), window, scale, padding)
        out["anchors"] = AnchorGenerator(api_utils.get_config()).generate_device((256, 256, 3)) \
            .cpu().numpy()

        overlays = visualize.composite_batch(eng, images, colors, annotate=True, class_names=NAMES)
        out["composite_batch"] = [o.cpu().numpy() for o in overlays]
        boxes = np.array([[4, 6, 30, 40], [10, 2, 50, 20]], np.int32)
        bmasks = gt_masks[0][:, :, :2]
        out["apply_masks"] = visualize.apply_masks(images[0], boxes, bmasks, colors[:2])
        out["encode_png"] = api_utils.encode_png_batch(images)
        out["encode_jpeg"] = api_utils.encode_jpeg_batch(images)
        return out


def _assert_same(a, b, where):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), where
        for k in a:
            _assert_same(a[k], b[k], f"{where}.{k}")
    elif isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f"{where}[{i}]")
    elif isinstance(a, np.ndarray):
        assert isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape, where
        assert a.tobytes() == b.tobytes(), where
    else:
        assert type(a) is type(b) and (a == b or a != a and b != b), where


def test_every_launch_runs_on_the_current_stream(recorder):
    import torch

    want = _workload(None)
    default_calls, recorder.calls = recorder.calls, []
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    got = _workload(s)
    torch.cuda.synchronize()
    names = {name for name, _ in recorder.calls}
    assert FAMILIES <= names, sorted(FAMILIES - names)
    assert names == {name for name, _ in default_calls}
    wrong = sorted({name for name, h in recorder.calls if h != s.cuda_stream})
    assert not wrong, f"launched off the current stream: {wrong}"
    _assert_same(got, want, "out")


def test_on_stream_enters_only_a_stream_not_current(cuda_device):
    """The pipeline launches' context: torch.cuda.stream(s) while s is not current, none when it
    is or when no stream is given; stream_ptr() is the current stream's handle throughout."""
    import torch

    s = torch.cuda.Stream()
    default = torch.cuda.current_stream()
    assert N.stream_ptr().value == (default.cuda_stream or None)
    ctx = N.on_stream(s)
    assert not isinstance(ctx, contextlib.nullcontext)
    with ctx:
        assert torch.cuda.current_stream() == s
        assert N.stream_ptr().value == s.cuda_stream
        assert isinstance(N.on_stream(s), contextlib.nullcontext)
        assert isinstance(N.on_stream(None), contextlib.nullcontext)
        assert not isinstance(N.on_stream(default), contextlib.nullcontext)
        with N.on_stream(default):
            assert torch.cuda.current_stream() == default
            assert N.stream_ptr().value == (default.cuda_stream or None)
        assert torch.cuda.current_stream() == s
    assert torch.cuda.current_stream() == default
