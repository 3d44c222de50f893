"""The canvas in memory from mrx_device_alloc (compressible where the GPU grants it): the kernels
must write the same bytes there as into a plain torch buffer, torch must read and write it like
any other device tensor, and `release()` must hand it back to the driver."""
import ctypes as C

import numpy as np
import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200 import synth

from helpers import prepared_engine

pytestmark = pytest.mark.gpu

CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED = 107


def _compression_supported(device):
    cu = C.CDLL("libcuda.so.1")
    value = C.c_int(-1)
    assert cu.cuDeviceGetAttribute(C.byref(value), CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED,
                                   int(device.index)) == 0
    return value.value


def _bench_images():
    import bench

    return bench.make_bench_images(0), 100, 81


def _ragged_images():
    rng = np.random.default_rng(1333)
    ims = [synth.make_image(rng, (800, 1333), n, num_classes=81, max_instances=100)
           for n in (100, 61, 0, 17, 100, 3)]
    return ims, 100, 81


def test_canvas_is_compressed_where_the_device_offers_it(cuda_device):
    ims, R, classes = _ragged_images()
    eng = prepared_engine(ims[:2], R, classes, np.float32)
    assert eng.canvas_compressed == (_compression_supported(cuda_device) == 1)


@pytest.mark.parametrize("images", [_bench_images, _ragged_images], ids=["bench", "ragged_800x1333"])
def test_canvas_bytes_equal_a_plain_buffer(cuda_device, images):
    import torch

    ims, R, classes = images()
    eng = prepared_engine(ims, R, classes, np.float32)
    total = int(eng._offsets[len(ims)])
    plain = torch.full((total,), 7, dtype=torch.uint8, device=cuda_device)
    eng.d_canvas.fill_(7)
    eng.enqueue_expand()
    eng.enqueue_expand(canvas_ptr=plain.data_ptr())
    counts = eng.fetch_meta()[0]
    assert counts.sum() > 0
    for b in range(len(ims)):
        H, W = (int(v) for v in eng._geom_host[b][:2])
        o, n = int(eng._offsets[b]), H * W * int(counts[b])
        assert torch.equal(eng.d_canvas[o:o + n], plain[o:o + n]), f"image {b}"
        assert n == 0 or int(plain[o:o + n].max()) <= 1


def test_canvas_view_round_trips(cuda_device):
    import torch

    ims, R, classes = _ragged_images()
    eng = prepared_engine(ims, R, classes, np.float32)
    eng.enqueue_expand()
    counts = eng.fetch_meta()[0]
    rng = np.random.default_rng(5)
    for b in (0, 3):
        k = int(counts[b])
        H, W = (int(v) for v in eng._geom_host[b][:2])
        host = torch.from_numpy((rng.random((H, W, k)) < 0.03).astype(np.uint8))
        eng.canvas_view(b, k).copy_(host)
        assert torch.equal(eng.canvas_view(b, k).cpu(), host)
        dev = host.to(cuda_device) ^ 1
        eng.canvas_view(b, k).copy_(dev)
        assert torch.equal(eng.canvas_view(b, k), dev)


def test_release_returns_the_canvas_memory(cuda_device):
    import torch

    ims, R, classes = _ragged_images()
    eng = prepared_engine(ims, R, classes, np.float32)
    total = int(eng._offsets[len(ims)])
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info(cuda_device)[0]
    eng.release()
    assert torch.cuda.mem_get_info(cuda_device)[0] >= before + total
