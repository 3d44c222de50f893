"""The host half of the device JPEG encoder: refusals, buffer sizing and the worst-case file
bound, the header constants and the ABI argument checks (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

import jpeg_encode_oracle as O
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils
from matterport_maskrcnn_with_tensorflow_serving_b200 import jpeg_encode as je


@pytest.mark.parametrize("shape,dtype,what", [
    ((4, 4, 3), np.float32, "dtype"), ((4, 4, 3), np.uint16, "dtype"), ((4, 4), np.uint8, "shape"),
    ((4, 4, 3, 1), np.uint8, "shape"), ((4, 4, 4), np.uint8, "shape"),
    ((4, 4, 1), np.uint8, "shape"), ((0, 4, 3), np.uint8, "pixel"), ((4, 0, 3), np.uint8, "pixel"),
    ((65536, 4, 3), np.uint8, "over 65535"), ((4, 65536, 3), np.uint8, "over 65535")])
def test_refusals_name_the_image(shape, dtype, what):
    with pytest.raises(ValueError, match=f"image 1: .*{what}"):
        je.EncodePlan([((2, 2, 3), np.uint8), (shape, dtype)])


@pytest.mark.parametrize("quality", [-1, 101, 1000, 95.0, "95", True, None])
def test_quality_refused(quality):
    with pytest.raises(ValueError, match="quality"):
        je.EncodePlan([((2, 2, 3), np.uint8)], quality)
    with pytest.raises(ValueError, match="quality"):
        api_utils.encode_jpeg_batch([np.zeros((2, 2, 3), np.uint8)], quality)


def test_refusals_before_any_device_work():
    """A bad image or quality raises from the plan, before CUDA is touched (none is needed)."""
    with pytest.raises(ValueError, match="image 1"):
        api_utils.encode_jpeg_batch([np.zeros((2, 2, 3), np.uint8), np.zeros((2, 2), np.uint8)])
    with pytest.raises(ValueError, match="quality"):
        api_utils.encode_jpeg_batch([], quality=101)
    assert api_utils.encode_jpeg_batch([]) == []


def test_plan_layout():
    shapes = [(2, 3), (100, 50), (1, 1), (33, 17)]
    plan = je.EncodePlan([((h, w, 3), np.uint8) for h, w in shapes], 75, True)
    d = plan.desc
    nblk = [6 * -(-h // 16) * -(-w // 16) for h, w in shapes]
    assert list(d[:, je.D_NBLK]) == nblk
    assert list(d[:, je.D_BLK_OFF]) == list(np.cumsum([0] + nblk[:-1]))
    nbt = [-(-n // je.BLOCK_TILE) for n in nblk]
    assert list(d[:, je.D_NBT]) == nbt and plan.block_tiles == sum(nbt)
    nyt = [-(-je.data_bound(n) // je.BYTE_TILE) for n in nblk]
    assert list(d[:, je.D_NYT]) == nyt and plan.byte_tiles == sum(nyt)
    assert all(o % 16 == 0 for o in d[:, je.D_OUT_OFF])
    assert list(d[:, je.D_MCUX]) == [-(-w // 16) for _, w in shapes]
    assert list(d[:, je.D_MCUY]) == [-(-h // 16) for h, _ in shapes]
    assert plan.max_blocks == max(nblk) and plan.max_bytes == je.data_bound(max(nblk))
    assert (plan.min_side, plan.max_side) == (1, 100)
    assert (plan.quality, plan.optimize) == (75, True)
    plan.set_sources([16, 32, 48, 64])
    assert list(d[:, je.D_SRC]) == [16, 32, 48, 64]


def test_header_bound_is_the_standard_tables_header():
    """The standard tables hold the most values a baseline table can (12 DC, 162 AC symbols)."""
    _, e = O.encode(np.zeros((8, 8, 3), np.uint8))
    assert e.hdr == je.MAX_HEADER


@pytest.mark.parametrize("h,w", [(16, 16), (64, 48), (17, 33), (1, 1), (96, 128)])
@pytest.mark.parametrize("content", ["noise", "checker"])
def test_bound_holds_at_the_worst_case(h, w, content):
    """Noise and full-swing checkerboards at quality 100 (every divisor 8: the largest
    categories) with the standard tables, and many 0xFF bytes to stuff."""
    rng = np.random.default_rng(h * 1000 + w)
    if content == "noise":
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    else:
        yy, xx = np.mgrid[:h, :w]
        img = np.repeat((((yy + xx) & 1) * 255).astype(np.uint8)[..., None], 3, 2)
    nblk = je.blocks(h, w)
    for optimize in (False, True):
        data, e = O.encode(img, 100, optimize)
        assert e.coef.shape[0] == nblk
        assert e.bits <= nblk * je.MAX_BLOCK_BITS and e.bytes <= je.data_bound(nblk)
        assert len(data) <= je.file_bound(nblk)


def test_header_constants():
    assert N.MRX_JPEG_ENC_MAX_SIDE == je.MAX_SIDE == 65535
    assert N.MRX_JPEG_ENC_INFO_WORDS == je.INFO_WORDS
    names = ["BITS", "BYTES", "FF", "HDR", "FILE", "BLOCKS"]
    assert [getattr(N, f"MRX_JPEG_ENC_{n}") for n in names] == list(range(6))


def _args(**kw):
    buf = C.c_void_p(16)
    a = dict(d_desc=buf, B=1, quality=95, optimize=0, min_side=1, max_side=16, max_blocks=6,
             max_bytes=1250, blk_tiles=1, byte_tiles=1, word_count=320)
    a.update(kw)
    return list(a.values()) + [buf] * 10 + [None]


def test_abi_checks():
    lib = N.load()
    assert lib.mrx_jpeg_encode(*_args(d_desc=None)) == N.MRX_E_INVALID
    assert b"null pointer" in lib.mrx_last_error()
    for kw in [dict(B=-1), dict(B=N.MRX_MAX_BATCH + 1), dict(quality=-1), dict(quality=101),
               dict(optimize=2), dict(max_blocks=0), dict(max_bytes=0), dict(blk_tiles=0)]:
        assert lib.mrx_jpeg_encode(*_args(**kw)) == N.MRX_E_INVALID, kw
    assert lib.mrx_jpeg_encode(*_args(max_side=65536)) == N.MRX_E_UNSUPPORTED
    assert b"65535" in lib.mrx_last_error()
    assert lib.mrx_jpeg_encode(*_args(min_side=0)) == N.MRX_E_UNSUPPORTED
    assert lib.mrx_jpeg_encode(*_args(B=0)) == N.MRX_OK


@pytest.mark.parametrize("kw", [dict(image_format="gif"), dict(image_format="jpeg", quality=101)])
def test_do_inference_refuses_a_bad_format_before_the_rpc(kw):
    from matterport_maskrcnn_with_tensorflow_serving_b200 import serve

    with pytest.raises(ValueError, match="image_format|quality"):
        serve.do_inference_batch([np.zeros((4, 4, 3), np.uint8)], **kw)
