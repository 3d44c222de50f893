"""`anchors_kernel` (csrc/anchors.cu) against `oracle.get_anchors`, bit for bit: image shapes the
backbone strides do not divide (the last anchors of a level lie outside the image), anchor
strides above 1, ratios and scales whose square roots and quotients are not exact, three to
eight pyramid levels, more anchors than one trip of the grid-stride loop; the row count and
row order from a closed form that does not go through the oracle; the memo."""
import ctypes as C
import math

import numpy as np
import pytest

import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import AnchorGenerator
from matterport_maskrcnn_with_tensorflow_serving_b200.model_configs import MaskRCNNServingConfig

from preprocess_inputs import assert_same, grid_stride_cap, mismatch

pytestmark = pytest.mark.gpu


def _config(**kw):
    return type("Cfg", (MaskRCNNServingConfig,), kw)


CONFIGS = {
    "default": MaskRCNNServingConfig,
    "anchor_stride_2": _config(RPN_ANCHOR_STRIDE=2),
    "anchor_stride_3": _config(RPN_ANCHOR_STRIDE=3),
    "ratios_inexact": _config(RPN_ANCHOR_RATIOS=[0.3, 1, 3.7]),
    "one_ratio": _config(RPN_ANCHOR_RATIOS=[1.5]),
    "eight_ratios": _config(RPN_ANCHOR_RATIOS=[0.2, 0.3, 0.5, 0.75, 1, 1.5, 2.5, 3.7]),
    "scales_inexact": _config(RPN_ANCHOR_SCALES=(24, 48, 96, 192, 384)),
    "three_levels": _config(BACKBONE_STRIDES=[8, 16, 32], RPN_ANCHOR_SCALES=(48, 96, 192)),
    "eight_levels": _config(BACKBONE_STRIDES=[2, 4, 8, 16, 32, 64, 128, 256],
                            RPN_ANCHOR_SCALES=(8, 16, 32, 64, 128, 256, 512, 1024)),
}
# (2, 2) is the smallest shape mrx_anchors accepts; the two largest give more anchors than the
# launch has threads
SHAPES = [(64, 64), (65, 63), (100, 1000), (2, 2), (1030, 770), (4096, 4096), (2160, 3840)]
LARGE_CONFIGS = ("default", "anchor_stride_2", "ratios_inexact", "scales_inexact")
CASES = [(hw, name) for hw in SHAPES for name in CONFIGS
         if hw[0] * hw[1] < 4_000_000 or name in LARGE_CONFIGS]


def _row_count(hw, cfg):
    a, n = cfg.RPN_ANCHOR_STRIDE, len(cfg.RPN_ANCHOR_RATIOS)
    return sum(math.ceil(math.ceil(hw[0] / s) / a) * math.ceil(math.ceil(hw[1] / s) / a) * n
               for s in cfg.BACKBONE_STRIDES)


@pytest.mark.parametrize("hw,name", CASES, ids=lambda v: str(v))
def test_shapes_and_configs(cuda_device, hw, name):
    cfg = CONFIGS[name]
    shape = (hw[0], hw[1], 3)
    ref = oracle.get_anchors(shape, cfg)
    gen = AnchorGenerator(cfg)
    assert gen.count(shape) == ref.shape[0] == _row_count(hw, cfg)
    if hw == (4096, 4096) and name == "default":
        assert ref.shape[0] > grid_stride_cap(ctas_per_sm=16)
    assert_same(gen.get_anchors(shape), ref, f"{name} {hw}")


def _random_config(rng):
    n_levels = int(rng.integers(1, N.MRX_MAX_LEVELS + 1))
    n_ratios = int(rng.integers(1, N.MRX_MAX_RATIOS + 1))
    return _config(
        BACKBONE_STRIDES=[int(v) for v in rng.integers(3, 101, size=n_levels)],
        RPN_ANCHOR_SCALES=tuple(float(v) for v in rng.uniform(4, 600, size=n_levels)),
        RPN_ANCHOR_RATIOS=[float(v) for v in rng.uniform(0.1, 5, size=n_ratios)],
        RPN_ANCHOR_STRIDE=int(rng.integers(1, 4)))


def test_seeded_sweep(cuda_device):
    rng = np.random.default_rng(41)
    failed = []
    for _ in range(60):
        cfg = _random_config(rng)
        hw = tuple(int(v) for v in rng.integers(2, 701, size=2))
        ref = oracle.get_anchors((hw[0], hw[1], 3), cfg)
        got = AnchorGenerator(cfg).get_anchors((hw[0], hw[1], 3))
        msg = mismatch(got, ref)
        if msg or ref.shape[0] != _row_count(hw, cfg):
            failed.append(f"{hw} strides {cfg.BACKBONE_STRIDES} scales {cfg.RPN_ANCHOR_SCALES} "
                          f"ratios {cfg.RPN_ANCHOR_RATIOS} stride {cfg.RPN_ANCHOR_STRIDE}: {msg}")
    assert not failed, f"{len(failed)} of 60 draws differ:\n" + "\n".join(failed[:10])


def _closed_form_row(hw, cfg, level, y, x, r):
    """Anchor (level, y, x, ratio r) in float64, rounded once to float32."""
    s, a = cfg.BACKBONE_STRIDES[level], cfg.RPN_ANCHOR_STRIDE
    scale, root = cfg.RPN_ANCHOR_SCALES[level], math.sqrt(cfg.RPN_ANCHOR_RATIOS[r])
    cy, cx, h, w = y * a * s, x * a * s, scale / root, scale * root
    box = [(cy - 0.5 * h) / (hw[0] - 1), (cx - 0.5 * w) / (hw[1] - 1),
           (cy + 0.5 * h - 1) / (hw[0] - 1), (cx + 0.5 * w - 1) / (hw[1] - 1)]
    return np.array(box, dtype=np.float64).astype(np.float32)


@pytest.mark.parametrize("hw,name", [((1030, 770), "ratios_inexact"), ((65, 63), "eight_ratios"),
                                     ((100, 1000), "anchor_stride_3"),
                                     ((2160, 3840), "scales_inexact")], ids=lambda v: str(v))
def test_row_order(cuda_device, hw, name):
    """Rows run level -> y -> x -> ratio: the first and last row of every level and rows drawn
    inside it equal the closed form of their (level, y, x, ratio)."""
    cfg = CONFIGS[name]
    got = AnchorGenerator(cfg).get_anchors((hw[0], hw[1], 3))
    assert got.shape == (_row_count(hw, cfg), 4) and got.dtype == np.float32
    a, n = cfg.RPN_ANCHOR_STRIDE, len(cfg.RPN_ANCHOR_RATIOS)
    rng = np.random.default_rng(42)
    off = 0
    for level, s in enumerate(cfg.BACKBONE_STRIDES):
        ny, nx = math.ceil(math.ceil(hw[0] / s) / a), math.ceil(math.ceil(hw[1] / s) / a)
        picks = [(0, 0, 0), (ny - 1, nx - 1, n - 1), (0, nx - 1, 0), (ny - 1, 0, n - 1)]
        picks += [(int(rng.integers(ny)), int(rng.integers(nx)), int(rng.integers(n)))
                  for _ in range(8)]
        for y, x, r in picks:
            row = off + (y * nx + x) * n + r
            assert_same(got[row], _closed_form_row(hw, cfg, level, y, x, r),
                        f"row {row} = level {level}, y {y}, x {x}, ratio {r}")
        off += ny * nx * n
    assert off == got.shape[0]


def _abi_counts(hw, strides, n_ratios, anchor_stride=1):
    out = C.c_longlong(-1)
    rc = N.load().mrx_anchor_count(hw[0], hw[1], N.int_array(strides), len(strides), n_ratios,
                                   anchor_stride, C.byref(out))
    return rc, out.value


def test_refusals(cuda_device):
    """Nine levels, nine ratios: outside what the kernel's parameter block holds.  A one-pixel
    side divides by h - 1 = 0 upstream."""
    import torch

    strides = [2, 4, 8, 16, 32, 64, 128, 256, 512]
    assert len(strides) == N.MRX_MAX_LEVELS + 1
    assert _abi_counts((64, 64), strides, 3) == (N.MRX_E_UNSUPPORTED, -1)
    assert _abi_counts((64, 64), strides[:8], 3)[0] == N.MRX_OK
    assert _abi_counts((64, 64), strides[:5], N.MRX_MAX_RATIOS + 1) == (N.MRX_E_UNSUPPORTED, -1)
    assert _abi_counts((64, 64), strides[:5], 0) == (N.MRX_E_UNSUPPORTED, -1)
    assert _abi_counts((64, 64), strides[:5], 3, anchor_stride=0) == (N.MRX_E_INVALID, -1)
    for hw in ((1, 1), (1, 64), (64, 1)):
        assert _abi_counts(hw, strides[:5], 3) == (N.MRX_E_INVALID, -1)
    nine = _config(RPN_ANCHOR_RATIOS=[0.2, 0.3, 0.5, 0.75, 1, 1.5, 2.5, 3.7, 4.0])
    with pytest.raises(N.MrxError):
        AnchorGenerator(nine).get_anchors((64, 64, 3))
    with pytest.raises(N.MrxError):
        AnchorGenerator(MaskRCNNServingConfig).get_anchors((1, 1, 3))
    # mrx_anchors itself, not only the count in front of it
    out = torch.full((15, 4), -7.0, dtype=torch.float32, device=cuda_device)
    cfg = MaskRCNNServingConfig
    rc = N.load().mrx_anchors(out, 1, 1, N.double_array(cfg.RPN_ANCHOR_SCALES),
                              N.double_array(cfg.RPN_ANCHOR_RATIOS),
                              N.int_array(cfg.BACKBONE_STRIDES), 5, 3, 1, N.stream_ptr(None))
    torch.cuda.synchronize()
    assert rc == N.MRX_E_INVALID and bool((out == -7.0).all())


# (side, scale): with one ratio of 1.0 the first anchor has y1 = x1 = -0.5 * scale exactly, and
# these scales put y1 / (side - 1) in float64 exactly half way between two float32 values just
# below 2, where y1 * (1 / (side - 1)) lands one float64 ulp to the side and rounds the other way
TIES = [(50, 195.99997079372406), (50, 195.9999941587448), (100, 395.999964594841)]


@pytest.mark.parametrize("side,scale", TIES, ids=str)
def test_division_not_reciprocal(cuda_device, side, scale):
    """norm_boxes divides.  A quotient on a float32 rounding tie is the input that tells a
    division from a multiplication by the reciprocal, which random shapes meet about once in
    2^29 values."""
    y1, d = -0.5 * scale, float(side - 1)
    assert np.float32(y1 / d) != np.float32(y1 * (1.0 / d)), "the case has lost its teeth"
    cfg = _config(RPN_ANCHOR_RATIOS=[1.0], RPN_ANCHOR_SCALES=(scale,) * 5)
    shape = (side, side, 3)
    ref = oracle.get_anchors(shape, cfg)
    assert ref[0, 0] == ref[0, 1] == np.float32(y1 / d)
    got = AnchorGenerator(cfg).get_anchors(shape)
    assert_same(got, ref, f"side {side}, scale {scale!r}")
    assert_same(got[0], _closed_form_row((side, side), cfg, 0, 0, 0, 0), "first anchor")


def test_memo(cuda_device):
    """One entry per shape however the shape is spelled, and `api_utils.set_config` drops the
    memo: the same shape then gives the new config's anchors."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils

    gen = AnchorGenerator(CONFIGS["default"])
    shape = (192, 256, 3)
    a1 = gen.get_anchors(shape)
    assert_same(a1, oracle.get_anchors(shape, CONFIGS["default"]), "default config")
    assert gen.get_anchors(list(shape)) is a1
    assert gen.get_anchors(np.array(shape)) is a1
    assert gen.get_anchors(tuple(np.int64(v) for v in shape)) is a1
    assert len(gen._cache) == 1
    assert gen.get_anchors((256, 192, 3)) is not a1 and len(gen._cache) == 2
    saved = api_utils.get_config()
    try:
        before = api_utils.get_anchors(shape)
        assert api_utils.get_anchors(list(shape)) is before
        assert_same(before, oracle.get_anchors(shape, saved), "configured anchors")
        api_utils.set_config(CONFIGS["ratios_inexact"]())
        after = api_utils.get_anchors(shape)
        assert after.shape == before.shape and not np.array_equal(after, before)
        assert_same(after, oracle.get_anchors(shape, CONFIGS["ratios_inexact"]), "after set_config")
    finally:
        api_utils.set_config(saved)
