"""Inputs shared by the pre-processing tests (test_gpu_cv2_resize / test_gpu_mold /
test_gpu_anchors): image makers, the (src, dst) pairs of `cv2.resize`, and the bit-for-bit
comparison every one of those tests ends in.

The image kinds are the ones on which a resize kernel's exactness claim can break.  Constant
and 0/255 images put every interpolated sample on or within an ulp of an integer, so a fused
multiply-add or a reassociated sum changes the truncated uint8; uniform noise reaches every
value of every weight; ramps make a transposed or shifted tap visible."""
import numpy as np

from matterport_maskrcnn_with_tensorflow_serving_b200 import synth


def noise(rng, h, w):
    return rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)


def checker(rng, h, w):
    """Every sample 0 or 255, drawn independently."""
    return (rng.integers(0, 2, size=(h, w, 3), dtype=np.uint8) * 255).astype(np.uint8)


def constant(value):
    def make(rng, h, w):
        return np.full((h, w, 3), value, dtype=np.uint8)
    make.__name__ = f"c{value}"
    return make


def ramp_h(rng, h, w):
    """Value grows along x (wrapping at 256), offset per channel."""
    row = (np.arange(w)[:, None] + np.array([0, 85, 170])) % 256
    return np.ascontiguousarray(np.broadcast_to(row[None], (h, w, 3)), dtype=np.uint8)


def ramp_v(rng, h, w):
    col = (np.arange(h)[:, None] + np.array([0, 85, 170])) % 256
    return np.ascontiguousarray(np.broadcast_to(col[:, None], (h, w, 3)), dtype=np.uint8)


KINDS = {"noise": noise, "checker": checker, "ramp_h": ramp_h, "ramp_v": ramp_v,
         "synth": synth.synth_rgb_image,
         **{f"c{v}": constant(v) for v in (0, 1, 127, 254, 255)}}


def make_image(kind, rng, h, w):
    img = KINDS[kind](rng, h, w)
    assert img.dtype == np.uint8 and img.shape == (h, w, 3) and img.flags.c_contiguous
    return img


# (source (h, w), destination (h, w)) at every branch decision of cv2.resize(INTER_LINEAR) on
# uint8: the exact-2x area shortcut and its near misses, identity, one-pixel sides (every tap
# clamped), large up- and down-scales
EDGE_PAIRS = [
    # exact 2x on both axes: the INTER_AREA box average
    ((2, 2), (1, 1)), ((6, 10), (3, 5)), ((1280, 1280), (640, 640)),
    ((1282, 1278), (641, 639)),
    # 2x on one axis only, 4x and 3x on both: integer scales that stay linear
    ((640, 1280), (640, 640)), ((1280, 640), (640, 640)),
    ((2560, 2560), (640, 640)), ((1920, 1920), (640, 640)),
    # 2x plus and minus a pixel
    ((1281, 1281), (640, 640)), ((1279, 1279), (640, 640)), ((1281, 1280), (640, 640)),
    # identity
    ((640, 640), (640, 640)), ((37, 91), (37, 91)),
    # one-pixel sides
    ((1, 1), (64, 64)), ((1, 1), (1, 1)), ((1, 500), (64, 48)), ((500, 1), (48, 64)),
    ((480, 640), (1, 1)), ((7, 9), (1, 1)), ((480, 640), (1, 333)), ((480, 640), (333, 1)),
    # scales above 100 and above 7
    ((3, 3), (640, 640)), ((2000, 3), (640, 640)), ((5000, 5000), (640, 640)),
]


def resize_pairs(seed, n_small=300, n_large=30):
    """EDGE_PAIRS (the small ones) followed by seeded random pairs: n_small with all four sides
    in [1, 200], n_large with one side, chosen at random, in [600, 2200]."""
    rng = np.random.default_rng(seed)
    pairs = [p for p in EDGE_PAIRS if max(p[0] + p[1]) <= 2200]
    for _ in range(n_small):
        s = rng.integers(1, 201, size=4)
        pairs.append(((int(s[0]), int(s[1])), (int(s[2]), int(s[3]))))
    for _ in range(n_large):
        s = rng.integers(1, 201, size=4)
        s[rng.integers(0, 4)] = rng.integers(600, 2201)
        pairs.append(((int(s[0]), int(s[1])), (int(s[2]), int(s[3]))))
    return pairs


def _bits(a):
    if a.dtype.kind == "f":
        return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])
    return a


def mismatch(got, ref):
    """None when `got` equals `ref` bit for bit (dtype and shape included), else a sentence
    with the number of differing elements, the first differing index and both values there."""
    got, ref = np.asarray(got), np.asarray(ref)
    if got.dtype != ref.dtype or got.shape != ref.shape:
        return f"got {got.dtype}{got.shape}, want {ref.dtype}{ref.shape}"
    g, r = _bits(np.ascontiguousarray(got)), _bits(np.ascontiguousarray(ref))
    if np.array_equal(g, r):
        return None
    bad = np.flatnonzero(g.reshape(-1) != r.reshape(-1))
    idx = tuple(int(v) for v in np.unravel_index(bad[0], got.shape))
    return (f"{bad.size} of {got.size} elements differ; first at {idx}: "
            f"got {got[idx]!r}, want {ref[idx]!r}")


def assert_same(got, ref, what):
    msg = mismatch(got, ref)
    assert msg is None, f"{what}: {msg}"


def grid_stride_cap(ctas_per_sm=32, threads=256):
    """Elements one trip of a grid-stride loop covers on the current device: the kernels of
    mold.cu launch at most 32 CTAs of 256 threads per SM, anchors.cu at most 16."""
    import torch

    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return ctas_per_sm * sms * threads
