"""`mold_image_kernel` (csrc/mold.cu) against `oracle.resize_image` + `oracle.mold_image`, bit
for bit: the truncated uint8 image and the float64 / float32 molded tensors on the pixels that
pin the operation order (constant, 0/255, noise, ramps), every resize mode and scalar of the
config that reaches the kernel, the batch entry point against the single-image one, the
refusals of the C ABI, and `serve.preprocess_input[_batch]` on the same pixels."""
import numpy as np
import pytest

import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import serve
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import Molder
from matterport_maskrcnn_with_tensorflow_serving_b200.model_configs import MaskRCNNServingConfig

from preprocess_inputs import assert_same, grid_stride_cap, make_image

pytestmark = pytest.mark.gpu

# upscale; downscale by IMAGE_MAX_DIM; scale 1 with and without padding; one- and two-pixel sides
SHAPES = [(300, 200), (97, 333), (480, 640), (1500, 1100), (2160, 3840), (1025, 3), (5, 1030),
          (1024, 1023), (800, 1024), (1024, 1024), (1, 1), (2, 900), (801, 799)]
# shapes whose constant-255 reference holds 254s ((480, 640) scales by 1.6 and holds none)
HOLDS_254 = [(300, 200), (97, 333), (1500, 1100), (801, 799)]
MOLD_KINDS = ["c255", "c1", "checker", "noise", "ramp_h", "ramp_v"]


def _oracle_mold(cfg, img):
    u8, window, scale, padding, _ = oracle.resize_image(
        img, min_dim=cfg.IMAGE_MIN_DIM, max_dim=cfg.IMAGE_MAX_DIM, min_scale=cfg.IMAGE_MIN_SCALE,
        mode=cfg.IMAGE_RESIZE_MODE)
    molded = oracle.mold_image(u8, cfg)
    assert molded.dtype == np.float64
    return u8, molded, window, scale, padding


def _same_scalars(got, ref, what):
    """Equal with Python `==` and of equal types, element by element: upstream packs window
    and scale into `image_meta`, whose dtype follows from them."""
    assert got == ref and type(got) is type(ref), (what, got, ref)
    if isinstance(ref, (tuple, list)):
        for g, r in zip(got, ref):
            _same_scalars(g, r, what)


def _check_mold(cfg, img, what):
    import torch

    ref_u8, ref_molded, window, scale, padding = _oracle_mold(cfg, img)
    m = Molder(cfg)
    d_img = torch.from_numpy(img).cuda()
    d64, u8, win, sc, pad = m.mold_device(d_img, np.float64, want_u8=True)
    _same_scalars(win, window, f"{what} window")
    _same_scalars(sc, scale, f"{what} scale")
    _same_scalars(pad, padding, f"{what} padding")
    assert_same(u8.cpu().numpy(), ref_u8, f"{what} uint8")
    assert_same(d64.cpu().numpy(), ref_molded, f"{what} float64")
    d32, u8b, _, _, _ = m.mold_device(d_img, np.float32, want_u8=True)
    assert_same(u8b.cpu().numpy(), ref_u8, f"{what} uint8 beside float32")
    assert_same(d32.cpu().numpy(), ref_molded.astype(np.float32), f"{what} float32")
    d32, none, _, _, _ = m.mold_device(d_img, np.float32)
    assert none is None
    assert_same(d32.cpu().numpy(), ref_molded.astype(np.float32), f"{what} float32 alone")
    return ref_u8


@pytest.mark.parametrize("kind", MOLD_KINDS)
@pytest.mark.parametrize("hw", SHAPES, ids=str)
def test_adversarial_pixels(cuda_device, hw, kind):
    img = make_image(kind, np.random.default_rng(21), *hw)
    ref_u8 = _check_mold(MaskRCNNServingConfig, img, f"{kind} {hw}")
    if kind == "c255" and hw in HOLDS_254:
        # the four weights do not always sum to 1 in scipy's order: samples just below 255
        # truncate to 254, and flip if one product is fused or the sum reassociated
        assert (ref_u8 == 254).any(), "the constant-255 reference holds no 254"


def _config(**kw):
    return type("Cfg", (MaskRCNNServingConfig,), kw)


CONFIGS = {
    # nothing scaled, padded by 61 = 30 + 31 rows and 59 = 29 + 30 columns
    "pad64_128_unscaled": (_config(IMAGE_RESIZE_MODE="pad64", IMAGE_MIN_DIM=128), (131, 197)),
    "pad64_128_scaled": (_config(IMAGE_RESIZE_MODE="pad64", IMAGE_MIN_DIM=128), (100, 333)),
    "pad64_128_exact": (_config(IMAGE_RESIZE_MODE="pad64", IMAGE_MIN_DIM=128), (128, 192)),
    # 512 x 765, padded by 3 = 1 + 2 columns
    "pad64_512_odd": (_config(IMAGE_RESIZE_MODE="pad64", IMAGE_MIN_DIM=512), (301, 450)),
    "pad64_512_even": (_config(IMAGE_RESIZE_MODE="pad64", IMAGE_MIN_DIM=512), (300, 451)),
    "none": (_config(IMAGE_RESIZE_MODE="none"), (123, 457)),
    "min_scale_2": (_config(IMAGE_MIN_SCALE=2.0), (450, 500)),
    "min_dim_0_small": (_config(IMAGE_MIN_DIM=0), (300, 200)),
    "min_dim_0_large": (_config(IMAGE_MIN_DIM=0), (1500, 1100)),
    "max_dim_2048": (_config(IMAGE_MIN_DIM=1600, IMAGE_MAX_DIM=2048), (480, 640)),
    # not exact in float32: the float32 output is the float64 difference rounded once
    "mean_pixel": (_config(MEAN_PIXEL=np.array([0.1, 1 / 3, 255.5])), (480, 640)),
    "mean_pixel_list": (_config(MEAN_PIXEL=[0.1, 1 / 3, 255.5]), (97, 333)),
}


@pytest.mark.parametrize("kind", ["noise", "c255"])
@pytest.mark.parametrize("name", CONFIGS)
def test_configs(cuda_device, name, kind):
    cfg, hw = CONFIGS[name]
    img = make_image(kind, np.random.default_rng(22), *hw)
    ref_u8 = _check_mold(cfg, img, f"{name} {kind} {hw}")
    if name == "max_dim_2048":   # 4.2 M pixels: the grid-stride loop's second trip
        assert ref_u8.shape[0] * ref_u8.shape[1] > grid_stride_cap()
    if name == "pad64_128_unscaled":
        assert ref_u8.shape == (192, 256, 3)
    if name == "pad64_512_odd":
        assert ref_u8.shape == (512, 768, 3)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("hw", [(97, 133), (1100, 1300)], ids=str)
@pytest.mark.parametrize("B", [1, 5, 33])
def test_batch_equals_single(cuda_device, B, hw, dtype):
    import torch

    rng = np.random.default_rng(23)
    imgs = np.stack([make_image("noise", rng, *hw) for _ in range(B)])
    m = Molder(MaskRCNNServingConfig)
    d_imgs = torch.from_numpy(imgs).cuda()
    out, window, scale, padding = m.mold_batch_device(d_imgs, dtype)
    assert out.shape[0] == B
    for b in range(B):
        one, _, win, sc, pad = m.mold_device(d_imgs[b], dtype)
        assert (win, sc, pad) == (window, scale, padding)
        if not torch.equal(out[b], one):
            assert_same(out[b].cpu().numpy(), one.cpu().numpy(), f"image {b} of {B}, {hw}")


def _mold_args(device, B, hw=(97, 133), dtype=np.float64):
    """Arguments of mrx_mold_image_batch for the default config on B noise images, with
    sentinel-filled outputs."""
    import torch

    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import resize_image_geometry

    cfg = MaskRCNNServingConfig
    rng = np.random.default_rng(24)
    imgs = np.stack([make_image("noise", rng, *hw) for _ in range(max(B, 1))])
    nh, nw, top, left, oh, ow, _, _, _ = resize_image_geometry(
        hw[0], hw[1], cfg.IMAGE_MIN_DIM, cfg.IMAGE_MAX_DIM, cfg.IMAGE_MIN_SCALE,
        cfg.IMAGE_RESIZE_MODE)
    tdtype = torch.float64 if dtype == np.float64 else torch.float32
    out = torch.full((max(B, 1), oh, ow, 3), -7.0, dtype=tdtype, device=device)
    u8 = torch.full((max(B, 1), oh, ow, 3), 0xA5, dtype=torch.uint8, device=device)
    geom = dict(src_h=hw[0], src_w=hw[1], new_h=nh, new_w=nw, top=top, left=left, out_h=oh,
                out_w=ow)
    return torch.from_numpy(imgs).to(device), geom, out, u8


def _call_mold_batch(d_imgs, B, geom, mean, code, out, u8):
    g = geom
    return N.load().mrx_mold_image_batch(
        d_imgs, B, g["src_h"], g["src_w"], g["new_h"], g["new_w"], g["top"], g["left"],
        g["out_h"], g["out_w"], mean, code, out, u8, N.stream_ptr(None))


MEAN = [123.7, 116.8, 103.9]


def _untouched(out, u8):
    import torch

    torch.cuda.synchronize()
    return bool((out == -7.0).all()) and bool((u8 == 0xA5).all())


def test_abi_empty_batch_writes_nothing(cuda_device):
    d_imgs, geom, out, u8 = _mold_args(cuda_device, 0)
    rc = _call_mold_batch(d_imgs, 0, geom, N.double_array(MEAN), N.MRX_F64, out, u8)
    assert rc == N.MRX_OK and _untouched(out, u8)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_abi_batch_with_uint8_output(cuda_device, dtype):
    """`d_molded_u8` of the batch entry: image b's truncated pixels land in slot b."""
    import torch

    B = 4
    d_imgs, geom, out, u8 = _mold_args(cuda_device, B, dtype=dtype)
    code = N.MRX_F64 if dtype == np.float64 else N.MRX_F32
    N.check(_call_mold_batch(d_imgs, B, geom, N.double_array(MEAN), code, out, u8),
            "mrx_mold_image_batch")
    torch.cuda.synchronize()
    for b in range(B):
        ref_u8, ref_molded, _, _, _ = _oracle_mold(MaskRCNNServingConfig, d_imgs[b].cpu().numpy())
        assert_same(u8[b].cpu().numpy(), ref_u8, f"uint8 of image {b}")
        assert_same(out[b].cpu().numpy(), ref_molded.astype(dtype), f"molded image {b}")


@pytest.mark.parametrize("case", ["too tall", "too wide", "negative top", "negative left",
                                  "out_dtype", "null mean", "null source", "null output",
                                  "new_h=0", "B=65536"])
def test_abi_refusals(cuda_device, case):
    d_imgs, geom, out, u8 = _mold_args(cuda_device, 2)
    B, code, mean = 2, N.MRX_F64, N.double_array(MEAN)
    src, dst = d_imgs, out
    if case == "too tall":
        geom["top"] = geom["out_h"] - geom["new_h"] + 1
    elif case == "too wide":
        geom["left"] = geom["out_w"] - geom["new_w"] + 1
    elif case == "negative top":
        geom["top"] = -1
    elif case == "negative left":
        geom["left"] = -1
    elif case == "out_dtype":
        code = 7
    elif case == "null mean":
        mean = None
    elif case == "null source":
        src = None
    elif case == "null output":
        dst = None
    elif case == "new_h=0":
        geom["new_h"] = 0
    elif case == "B=65536":
        B = 65536
    assert _call_mold_batch(src, B, geom, mean, code, dst, u8) == N.MRX_E_INVALID, case
    if case != "B=65536":   # the single-image entry takes the same checks
        g = geom
        rc = N.load().mrx_mold_image(
            src, g["src_h"], g["src_w"], g["new_h"], g["new_w"], g["top"], g["left"],
            g["out_h"], g["out_w"], mean, code, dst, u8, N.stream_ptr(None))
        assert rc == N.MRX_E_INVALID, case
    assert _untouched(out, u8)


def _same_preprocessed(got, ref, what):
    molded, meta, anchors, window = got
    ref_molded, ref_meta, ref_anchors, ref_window = ref
    assert window == ref_window, what
    assert_same(molded, ref_molded, f"{what} molded")
    assert_same(meta, ref_meta, f"{what} image_meta")
    assert_same(anchors, ref_anchors, f"{what} anchors")


@pytest.mark.parametrize("kind", ["c255", "checker", "noise"])
@pytest.mark.parametrize("img_size", [640, 1024, 320, None])
def test_preprocess_input(cuda_device, img_size, kind):
    img = make_image(kind, np.random.default_rng(25), 480, 640)
    _same_preprocessed(serve.preprocess_input(img, img_size),
                       oracle.preprocess_input(img, img_size), f"{kind} {img_size}")


@pytest.mark.parametrize("img_size", [640, 1024, 320, None])
def test_preprocess_input_batch(cuda_device, img_size):
    """Images of mixed sizes and kinds, one of them a view with a negative and a non-unit
    stride: the host packing must not depend on contiguity."""
    rng = np.random.default_rng(26)
    view = make_image("noise", rng, 600, 800)[::-1, ::2]
    assert view.shape == (600, 400, 3) and not view.flags.c_contiguous and view.strides[0] < 0
    if img_size is None:    # one size for all
        imgs = [make_image("c255", rng, 600, 400), view, make_image("checker", rng, 600, 400)]
    else:
        imgs = [make_image("noise", rng, 1, 1), make_image("checker", rng, 1280, 1280), view,
                make_image("c255", rng, 97, 333), make_image("noise", rng, 1280, 1280)]
    molded, metas, anchors, windows = serve.preprocess_input_batch(imgs, img_size, np.float64)
    m32, metas32, _, _ = serve.preprocess_input_batch(imgs, img_size)
    for b, img in enumerate(imgs):
        ref = oracle.preprocess_input(np.ascontiguousarray(img), img_size)
        _same_preprocessed((molded[b], metas[b], anchors, windows[b]), ref,
                           f"image {b} at {img_size}")
        assert_same(m32[b], ref[0].astype(np.float32), f"image {b} at {img_size}, float32")
        assert_same(metas32[b], ref[1], f"image {b} at {img_size}, image_meta beside float32")
        _same_preprocessed(serve.preprocess_input(img, img_size), ref,
                           f"image {b} alone at {img_size}")
