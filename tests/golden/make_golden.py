"""Generates tests/golden/*.npz from the oracle (run here, on CPU).  The reference ships
no fixtures for this path and its implementation is not importable (SURVEY.md 8c), so these
vectors pin the ORACLE (parity unpinned w.r.t. the reference itself): they catch drift of
the restatement and give the GPU tests small cases whose expected output is a committed
file rather than something recomputed at test time.

    python tests/golden/make_golden.py               # every file
    python tests/golden/make_golden.py jpeg_edges    # one of CASES
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from matterport_maskrcnn_with_tensorflow_serving_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def unmold_case(name, seed, hw, n, classes, R, **kw):
    rng = np.random.default_rng(seed)
    im = synth.make_image(rng, hw, n, num_classes=classes, max_instances=R, **kw)
    det = im.detections.astype(np.float64)
    msk = im.mrcnn_mask.astype(np.float64)
    b, c, s, m, rz = oracle.unmold_detections(det, msk, im.original_image_shape, im.image_shape,
                                              im.window, return_resized=True)
    band = np.zeros(m.shape, dtype=bool)     # pixels whose float64 value is within 1e-6 of 0.5
    for i, (y1, x1, y2, x2) in enumerate(b):
        band[y1:y2, x1:x2, i] = np.abs(rz[i] - 0.5) <= 1e-6
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        detections=im.detections, mrcnn_mask=im.mrcnn_mask,
        original_image_shape=np.array(im.original_image_shape),
        image_shape=np.array(im.image_shape), window=np.array(im.window),
        boxes=b, class_ids=c, scores=s,
        masks_packed=np.packbits(m, axis=None), masks_shape=np.array(m.shape),
        band_packed=np.packbits(band, axis=None))
    print(name, "N =", b.shape[0], "ones =", int(m.sum()), "band px =", int(band.sum()))


def anchors_case():
    out = {}
    for hw in [(64, 64), (256, 320), (512, 512), (1024, 1024), (800, 1344)]:
        a = oracle.get_anchors((hw[0], hw[1], 3))
        key = f"{hw[0]}x{hw[1]}"
        out[key + "_count"] = np.array(a.shape[0])
        out[key + "_sha256"] = np.frombuffer(hashlib.sha256(a.tobytes()).digest(), dtype=np.uint8)
        out[key + "_head"] = a[:6]
        out[key + "_tail"] = a[-6:]
    np.savez_compressed(os.path.join(HERE, "anchors.npz"), **out)
    print("anchors", {k: int(v) for k, v in out.items() if k.endswith("_count")})


def resize_case():
    rng = np.random.default_rng(42)
    tile = rng.random((28, 28), dtype=np.float32)
    out = {"tile": tile}
    for (bh, bw) in [(28, 28), (5, 9), (57, 31), (100, 37), (1, 1)]:
        out[f"out_{bh}x{bw}"] = oracle.resize(tile.astype(np.float64), (bh, bw))
    np.savez_compressed(os.path.join(HERE, "resize.npz"), **out)


def composite_case():
    """Overlay of display_instances (SURVEY.md 8f rank 2) on the unmold_small masks."""
    import random

    g = np.load(os.path.join(HERE, "unmold_small.npz"))
    shape = tuple(int(v) for v in g["masks_shape"])
    masks = np.unpackbits(g["masks_packed"], count=int(np.prod(shape))).reshape(shape).astype(bool)
    rng = np.random.default_rng(7)
    image = synth.synth_rgb_image(rng, shape[0], shape[1])
    colors = oracle.random_colors(shape[2], rng=random.Random(11))
    out = oracle.composite_instances(image, g["boxes"], masks, colors, alpha=0.5)
    np.savez_compressed(os.path.join(HERE, "composite_small.npz"), image=image,
                        colors=np.array(colors, dtype=np.float64), overlay=out)
    print("composite_small", out.shape, "sha", hashlib.sha256(out.tobytes()).hexdigest()[:12])


def jpeg_edges_case():
    """tests/jpeg_edge_inputs.py's files (baseline and progressive) with cv2.imdecode's decode of
    each: the array when it is small, else its shape and SHA-256; plus the SHA-256 of the three
    full 2048 x 2048 colour grids, and the cv2 / libjpeg-turbo versions and CPU that made them."""
    import platform
    import re

    import cv2

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import jpeg_edge_inputs as E
    import jpeg_inputs as JI

    base = E.all_cases()
    cases = base + E.progressive(base)
    blobs = [c.blob for c in cases]
    out = {"names": np.array([c.name for c in cases]),
           "files": np.frombuffer(b"".join(blobs), dtype=np.uint8),
           "file_off": np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64),
           "file_sha256": np.array([hashlib.sha256(b).hexdigest() for b in blobs])}
    ok, shape, sha = [], [], []
    for c in cases:
        img = JI.cv2_decode(c.blob)
        ok.append(img is not None)
        shape.append(img.shape if img is not None else (0, 0, 0))
        sha.append(hashlib.sha256(img.tobytes()).hexdigest() if img is not None else "")
        if img is not None and img.size <= 3 * 64 * 64:
            out["px_" + c.name] = img
    out.update(cv2_ok=np.array(ok), shape=np.array(shape, dtype=np.int64), px_sha256=np.array(sha))
    for c in E.colour_grids(step=1):
        img = JI.cv2_decode(c.blob)
        out["grid_sha256_" + c.name] = np.array(hashlib.sha256(img.tobytes()).hexdigest())
    info = cv2.getBuildInformation()
    turbo = re.search(r"JPEG:\s+\S+ \(ver ([^)]*)\)", info)
    with open("/proc/cpuinfo") as f:
        avx2 = " avx2" in f.read()
    out.update(cv2_version=np.array(cv2.__version__),
               libjpeg_turbo_version=np.array(turbo.group(1) if turbo else "unknown"),
               cpu=np.array(platform.machine() + (" avx2" if avx2 else "")))
    np.savez_compressed(os.path.join(HERE, "jpeg_edges.npz"), **out)
    print("jpeg_edges", len(cases), "files,", int(out["file_off"][-1]), "bytes;",
          str(out["cv2_version"]), str(out["libjpeg_turbo_version"]), str(out["cpu"]))


CASES = {"unmold": lambda: (unmold_case("unmold_small", 101, (96, 128), 12, 5, 16,
                                        zero_area_rows=(3,)),
                            unmold_case("unmold_coco_shape", 102, (120, 200), 9, 4, 12)),
         "anchors": anchors_case, "resize": resize_case, "composite": composite_case,
         "jpeg_edges": jpeg_edges_case}


if __name__ == "__main__" and len(sys.argv) > 1:    # python make_golden.py jpeg_edges ...
    for name in sys.argv[1:]:
        CASES[name]()
elif __name__ == "__main__":
    unmold_case("unmold_small", 101, (96, 128), 12, 5, 16, zero_area_rows=(3,))
    unmold_case("unmold_coco_shape", 102, (120, 200), 9, 4, 12)
    anchors_case()
    resize_case()
    composite_case()
    jpeg_edges_case()
