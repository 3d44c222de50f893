"""The device PNG encoder (csrc/png.cu) on the edge images of tests/png_encode_edge_inputs.py:
files equal to cv2.imencode('.png') byte for byte through encode_png_batch, from tensors and from
arrays, each image alone, first in a batch and in a later slot of a batch mixed with matrix
images; and the device's symbol and block counts, file size and per-block types, bit offsets and
bit lengths equal to the oracle's."""
import functools

import numpy as np
import pytest
import torch

import png_encode_edge_inputs as E
import png_inputs
import png_oracle as P
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, png

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")


@functools.lru_cache(maxsize=None)
def _cases():
    return E.all_cases()


@functools.lru_cache(maxsize=None)
def _ref(k):
    img = _cases()[k].img
    return cv2.imencode(".png", np.ascontiguousarray(img[..., ::-1]))[1].tobytes()


@functools.lru_cache(maxsize=None)
def _matrix():
    return [(name, img) for name, img in png_inputs.matrix(big=False)
            if name in ("noise2x2", "const1x7", "runs", "sym16383", "noise333x1")]


def _inputs(arrays, source, dev):
    return [torch.from_numpy(a).to(dev) for a in arrays] if source == "tensor" else arrays


def _mref(name, img):
    return cv2.imencode(".png", np.ascontiguousarray(img[..., ::-1]))[1].tobytes()


@pytest.mark.parametrize("source", ["tensor", "array"])
def test_each_edge_image_alone_and_first(cuda_device, source):
    name, other = _matrix()[0]
    for k, case in enumerate(_cases()):
        got = api_utils.encode_png_batch(_inputs([case.img], source, cuda_device))
        assert got == [_ref(k)], case.name
        got = api_utils.encode_png_batch(_inputs([case.img, other], source, cuda_device))
        assert got[0] == _ref(k) and got[1] == _mref(name, other), case.name


@pytest.mark.parametrize("source", ["tensor", "array"])
def test_mixed_batches_later_slots(cuda_device, source):
    """All edge images in one batch, each after a matrix image (so none but the first is in slot
    0), and the same batch in reverse order."""
    mats = _matrix()
    arrays, refs, names = [], [], []
    for k, case in enumerate(_cases()):
        mn, mi = mats[k % len(mats)]
        arrays += [mi, case.img]
        refs += [_mref(mn, mi), _ref(k)]
        names += [mn, case.name]
    for order in (slice(None), slice(None, None, -1)):
        got = api_utils.encode_png_batch(_inputs(arrays[order], source, cuda_device))
        for g, r, n in zip(got, refs[order], names[order]):
            assert g == r, n


def test_device_intermediates_equal_the_oracle(cuda_device):
    """NSYM, NBLK and FILE per image; TYPE, BITS and BIT per block."""
    cases = _cases()
    files, img_info, blk_info, plan = api_utils._png_encode([c.img for c in cases], stats=True)
    for b, case in enumerate(cases):
        data, e = P.encode(case.img)
        assert files[b] == data == _ref(b), case.name
        assert img_info[b, N.MRX_PNG_IMG_NSYM] == e.nsym, case.name
        assert img_info[b, N.MRX_PNG_IMG_NBLK] == len(e.blocks), case.name
        assert img_info[b, N.MRX_PNG_IMG_FILE] == len(data), case.name
        k0 = int(plan.desc[b, png.D_BLK_OFF])
        rows = blk_info[k0:k0 + len(e.blocks)]
        assert list(rows[:, N.MRX_PNG_BLK_TYPE]) == [blk.type for blk in e.blocks], case.name
        assert list(rows[:, N.MRX_PNG_BLK_BITS]) == [blk.bits for blk in e.blocks], case.name
        assert list(rows[:, N.MRX_PNG_BLK_BIT]) == [blk.bit_start for blk in e.blocks], case.name
