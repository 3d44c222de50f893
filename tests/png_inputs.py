"""The image matrix of the PNG encoder tests: sizes at the corners, on both sides of every window
bits boundary, a symbol count that is an exact multiple of 16383, chosen run lengths, constant,
noise, synthetic and overlay images, and 2160x3840."""
import random

import numpy as np

import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import synth


def image_from_stream(f, h, w):
    """The uint8 [h, w, 3] image whose filtered stream (Sub, w > 1) has the sample bytes f [h, 3w]."""
    f = np.asarray(f, dtype=np.uint8).reshape(h, 3 * w)
    raw = np.zeros_like(f)
    raw[:, :3] = f[:, :3]
    for x in range(3, 3 * w, 3):
        raw[:, x:x + 3] = f[:, x:x + 3] + raw[:, x - 3:x]
    return raw.reshape(h, w, 3)


def run_free_stream(rng, h, w):
    """Sample bytes with no byte equal to its predecessor in the filtered stream (filter byte 1
    at every row start): every position is its own literal."""
    f = rng.integers(0, 256, size=(h, 3 * w)).astype(np.int64)
    flat = np.concatenate([np.ones((h, 1), np.int64), f], axis=1).reshape(-1)
    for i in range(1, len(flat)):
        if i % (3 * w + 1) == 0:
            continue
        while flat[i] == flat[i - 1] or (i + 1 < len(flat) and (i + 1) % (3 * w + 1) == 0
                                          and flat[i] == 1):
            flat[i] = (flat[i] + 1) % 256
    return flat.reshape(h, 3 * w + 1)[:, 1:]


def runs_image(rng, h=24, w=120):
    """Runs of identical filtered bytes of 3, 4, 258, 259, 260, 261, 262 bytes, and runs of 1s
    that cross row boundaries through the filter byte."""
    f = run_free_stream(rng, h, w).reshape(-1).copy()
    pos = 5
    for length in (3, 4, 258, 259, 260, 261, 262, 3, 517, 775):
        v = int(rng.integers(2, 256))
        f[pos:pos + length] = v
        pos += length + 7
    row = 3 * w
    for r in (10, 15, 20):        # ... 1 1 1 | filter 1 | 1 1 ... across rows r-1 and r
        f[r * row - 4:r * row] = 1
        f[r * row:r * row + 3] = 1
    return image_from_stream(f, h, w)


def overlay(rng, h, w, n=6):
    """An overlay as display_instances makes it: oracle.composite_instances of box masks."""
    image = synth.synth_rgb_image(rng, h, w)
    boxes = np.zeros((n, 4), np.int32)
    masks = np.zeros((h, w, n), bool)
    for i in range(n):
        y1, x1 = int(rng.integers(0, h)), int(rng.integers(0, w))
        y2, x2 = int(rng.integers(y1, h)) + 1, int(rng.integers(x1, w)) + 1
        boxes[i] = (y1, x1, y2, x2)
        yy, xx = np.mgrid[y1:y2, x1:x2]
        cy, cx = (y1 + y2) / 2, (x1 + x2) / 2
        masks[y1:y2, x1:x2, i] = ((yy - cy) / max(y2 - y1, 1)) ** 2 + \
            ((xx - cx) / max(x2 - x1, 1)) ** 2 < 0.2
    colors = oracle.random_colors(n, rng=random.Random(int(rng.integers(1 << 30))))
    return oracle.composite_instances(image, boxes, masks, colors, alpha=0.5)


def matrix(big=True):
    """[(name, uint8 [H, W, 3] RGB image)]."""
    rng = np.random.default_rng(2024)
    out = []
    for h, w in [(1, 1), (1, 7), (9, 1), (2, 2)]:
        out.append((f"noise{h}x{w}", rng.integers(0, 256, (h, w, 3), dtype=np.uint8)))
        out.append((f"const{h}x{w}", np.full((h, w, 3), 200, np.uint8)))
    # n = 3W + 1 on both sides of each window bits boundary
    for bound in (16384, 8192, 4096, 2048, 1024, 512, 256, 128):
        for w in ((bound - 1) // 3, (bound - 1) // 3 + 1):
            out.append((f"wb{bound}_w{w}", synth.synth_rgb_image(rng, 1, w)))
    # 129 rows of 127 filtered bytes, none equal to its predecessor: 16383 symbols, so the final
    # block is empty; twice that for two full blocks
    out.append(("sym16383", image_from_stream(run_free_stream(rng, 129, 42), 129, 42)))
    out.append(("sym32766", image_from_stream(run_free_stream(rng, 258, 42), 258, 42)))
    out.append(("runs", runs_image(rng)))
    out.append(("const300x200", np.full((300, 200, 3), 7, np.uint8)))
    out.append(("noise300x200", rng.integers(0, 256, (300, 200, 3), dtype=np.uint8)))
    out.append(("noise333x1", rng.integers(0, 256, (333, 1, 3), dtype=np.uint8)))
    out.append(("synth240x320", synth.synth_rgb_image(rng, 240, 320)))
    out.append(("levels200x260", (rng.integers(0, 3, (200, 260, 3)) * 90).astype(np.uint8)))
    out.append(("overlay256x256", overlay(rng, 256, 256)))
    out.append(("overlay480x640", overlay(rng, 480, 640)))
    if big:
        out.append(("noise700x900", rng.integers(0, 256, (700, 900, 3), dtype=np.uint8)))
        out.append(("overlay2160x3840", overlay(rng, 2160, 3840, 12)))
    return out
