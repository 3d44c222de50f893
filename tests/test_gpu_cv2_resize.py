"""`cv2_resize_kernel` (csrc/mold.cu) against the real `cv2.resize`, bit for bit: every branch of
OpenCV's uint8 INTER_LINEAR (the exact-2x area shortcut and its near misses, one-pixel sides,
identity, scales above 100), a seeded sweep of sizes, destinations past one trip of the
grid-stride loop, the batch entry point slot by slot against the single-image one, the
refusals of the C ABI, and a source past 2^31 bytes."""
import math
import os

import numpy as np
import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import Molder
from matterport_maskrcnn_with_tensorflow_serving_b200.model_configs import MaskRCNNServingConfig

from preprocess_inputs import (EDGE_PAIRS, assert_same, grid_stride_cap, make_image, mismatch,
                               resize_pairs)

pytestmark = pytest.mark.gpu

GB = 1 << 30


def _cv2_resize(img, dst):
    import cv2

    return cv2.resize(img, (dst[1], dst[0]))


def _device_resize(img, dst):
    import torch

    m = Molder(MaskRCNNServingConfig)
    return m.cv2_resize_device(torch.from_numpy(img).cuda(), dst).cpu().numpy()


@pytest.mark.parametrize("kind", ["noise", "checker"])
@pytest.mark.parametrize("src,dst", EDGE_PAIRS, ids=lambda p: "x".join(map(str, p)))
def test_branch_pairs(cuda_device, src, dst, kind):
    """Each decision of cv::resize on both of its sides; 0/255 pixels are the only ones that
    reach the ends of the fixed-point range."""
    img = make_image(kind, np.random.default_rng(11), *src)
    assert_same(_device_resize(img, dst), _cv2_resize(img, dst), f"{kind} {src}->{dst}")


def test_seeded_sweep(cuda_device):
    pairs = resize_pairs(5)
    assert sum(max(s + d) <= 200 for s, d in pairs) >= 300
    assert sum(max(s + d) >= 600 for s, d in pairs) >= 30
    rng = np.random.default_rng(6)
    failed = []
    for src, dst in pairs:
        img = make_image("noise", rng, *src)
        msg = mismatch(_device_resize(img, dst), _cv2_resize(img, dst))
        if msg:
            failed.append(f"{src}->{dst}: {msg}")
    assert not failed, f"{len(failed)} of {len(pairs)} pairs differ:\n" + "\n".join(failed[:20])


@pytest.mark.parametrize("kind", ["noise", "checker"])
@pytest.mark.parametrize("dst", ["just_past", (2048, 2048), (1500, 3000)], ids=str)
def test_grid_stride_second_trip(cuda_device, dst, kind):
    """Destinations with more pixels than the launch has threads: the loop's stride is used."""
    cap = grid_stride_cap()
    if dst == "just_past":   # 1040 x 1040 on a 132-SM part
        dst = (math.isqrt(cap) + 1,) * 2
    assert dst[0] * dst[1] > cap, (dst, cap)
    img = make_image(kind, np.random.default_rng(12), 777, 1333)
    assert_same(_device_resize(img, dst), _cv2_resize(img, dst), f"{kind} ->{dst}")


# image 0 is the smallest of the list
BATCH_SIZES = [(1, 1), (1, 500), (500, 1), (7, 9), (480, 640), (1280, 1280), (2160, 3840),
               (333, 517), (333, 517)]


@pytest.mark.parametrize("dst", [(640, 640), (37, 91)], ids=str)
def test_batch_equals_single(cuda_device, dst):
    """One launch over nine slots of mixed sizes (the 1280^2 one takes the area shortcut at
    640^2, its neighbours the linear branch) equals, slot by slot, the single-image launch and
    cv2; the sources come back as they went in."""
    import torch

    rng = np.random.default_rng(13)
    imgs = [make_image("noise", rng, *hw) for hw in BATCH_SIZES]
    before = [im.copy() for im in imgs]
    m = Molder(MaskRCNNServingConfig)
    out, sources = m.cv2_resize_batch_device(imgs, dst, return_sources=True)
    assert out.shape == (len(imgs), dst[0], dst[1], 3) and out.dtype == torch.uint8
    assert_same(m.cv2_resize_batch_device(imgs, dst).cpu().numpy(), out.cpu().numpy(),
                "without return_sources")
    out = out.cpu().numpy()
    assert len(sources) == len(imgs)
    for b, img in enumerate(imgs):
        assert sources[b] is img
        assert_same(img, before[b], f"source {b}")
        assert_same(out[b], _device_resize(img, dst), f"slot {b} {img.shape[:2]} vs single")
        assert_same(out[b], _cv2_resize(img, dst), f"slot {b} {img.shape[:2]} vs cv2")


def _batch_args(device, B=2, dst=(8, 8)):
    import torch

    src = torch.zeros(64, dtype=torch.uint8, device=device)
    off = torch.tensor([0, 16], dtype=torch.int64, device=device)
    hw = torch.tensor([[2, 2], [2, 2]], dtype=torch.int32, device=device)
    out = torch.full((max(B, 1), dst[0], dst[1], 3), 0xA5, dtype=torch.uint8, device=device)
    return src, off, hw, out


def _untouched(out):
    import torch

    torch.cuda.synchronize()
    return bool((out == 0xA5).all())


def test_abi_empty_batch_writes_nothing(cuda_device):
    lib = N.load()
    src, off, hw, out = _batch_args(cuda_device)
    rc = lib.mrx_cv2_resize_u8c3_batch(src, off, hw, out, 0, 8, 8, N.stream_ptr(None))
    assert rc == N.MRX_OK and _untouched(out)


@pytest.mark.parametrize("case", ["B=65536", "dst_h=0", "dst_w=0", "null offsets", "null sizes",
                                  "null source", "null destination", "B=-1"])
def test_abi_batch_refusals(cuda_device, case):
    lib = N.load()
    src, off, hw, out = _batch_args(cuda_device)
    B, dh, dw = 2, 8, 8
    args = {"src": src, "off": off, "hw": hw, "out": out}
    if case == "B=65536":
        B = 65536
    elif case == "B=-1":
        B = -1
    elif case == "dst_h=0":
        dh = 0
    elif case == "dst_w=0":
        dw = 0
    else:
        args[{"null offsets": "off", "null sizes": "hw", "null source": "src",
              "null destination": "out"}[case]] = None
    rc = lib.mrx_cv2_resize_u8c3_batch(args["src"], args["off"], args["hw"], args["out"], B, dh,
                                       dw, N.stream_ptr(None))
    assert rc == N.MRX_E_INVALID, case
    assert _untouched(out)


@pytest.mark.parametrize("sizes", [(0, 4, 8, 8), (4, 0, 8, 8), (4, 4, 0, 8), (4, 4, 8, 0),
                                   (-1, 4, 8, 8)], ids=str)
def test_abi_single_refuses_empty_sides(cuda_device, sizes):
    lib = N.load()
    src, _, _, out = _batch_args(cuda_device)
    sh, sw, dh, dw = sizes
    rc = lib.mrx_cv2_resize_u8c3(src, sh, sw, out, dh, dw, N.stream_ptr(None))
    assert rc == N.MRX_E_INVALID and _untouched(out)


BIG = 27000          # 27000 x 27000 x 3 = 2.187e9 bytes, above 2^31 = 2.147e9


def _host_free_bytes():
    return os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")


def _big_source(nbytes_device):
    """The 27000^2 source, filled on the device from a seeded generator, inside a buffer of
    `nbytes_device` bytes at the offset that puts it last."""
    import torch

    n = BIG * BIG * 3
    assert n > 2 ** 31
    free = torch.cuda.mem_get_info()[0]
    if free < nbytes_device + GB:
        pytest.skip(f"needs {(nbytes_device + GB) / GB:.1f} GB of free device memory; "
                    f"{free / GB:.1f} GB are free")
    if _host_free_bytes() < n + 2 * GB:
        pytest.skip(f"needs {(n + 2 * GB) / GB:.1f} GB of free host memory for cv2's copy; "
                    f"{_host_free_bytes() / GB:.1f} GB are free")
    buf = torch.empty(nbytes_device, dtype=torch.uint8, device="cuda")
    big = buf[nbytes_device - n:].view(BIG, BIG, 3)
    g = torch.Generator(device="cuda").manual_seed(2031)
    for y in range(0, BIG, 1000):   # each fill stays below 2^31 elements
        big[y:y + 1000].random_(0, 256, generator=g)
    return buf, big


@pytest.mark.parametrize("through", ["single", "batch"])
def test_source_past_2g_bytes(cuda_device, through):
    """A 27000 x 27000 RGB source (2.19 GB; the JPEG decoder accepts headers up to 2^30 pixels)
    to 640^2 and 1024^2: byte offsets of the lower rows do not fit 32 bits.  Through the batch
    entry the image lies in the second slot, whose `src_off` is itself above 2^31."""
    import torch

    lib = N.load()
    n = BIG * BIG * 3
    if through == "single":
        buf, big = _big_source(n)
    else:
        off1 = 2 ** 31 + 16
        buf, big = _big_source(off1 + n)
        small = make_image("noise", np.random.default_rng(14), 48, 64)
        buf[:small.size] = torch.from_numpy(small).cuda().reshape(-1)
        d_off = torch.tensor([0, off1], dtype=torch.int64, device="cuda")
        d_hw = torch.tensor([[48, 64], [BIG, BIG]], dtype=torch.int32, device="cuda")
    host = big.cpu().numpy()
    assert host.nbytes == n > 2 ** 31
    for dst in ((640, 640), (1024, 1024)):
        ref = _cv2_resize(host, dst)
        if through == "single":
            out = torch.empty((dst[0], dst[1], 3), dtype=torch.uint8, device="cuda")
            N.check(lib.mrx_cv2_resize_u8c3(big, BIG, BIG, out, dst[0], dst[1],
                                            N.stream_ptr(None)), "mrx_cv2_resize_u8c3")
            assert_same(out.cpu().numpy(), ref, f"{BIG}^2 -> {dst}")
        else:
            out = torch.empty((2, dst[0], dst[1], 3), dtype=torch.uint8, device="cuda")
            N.check(lib.mrx_cv2_resize_u8c3_batch(buf, d_off, d_hw, out, 2, dst[0], dst[1],
                                                  N.stream_ptr(None)),
                    "mrx_cv2_resize_u8c3_batch")
            out = out.cpu().numpy()
            assert_same(out[0], _cv2_resize(small, dst), f"slot 0 -> {dst}")
            assert_same(out[1], ref, f"slot 1, {BIG}^2 at offset {off1} -> {dst}")
