"""The device JPEG decoder (csrc/jpeg.cu) against cv2.imdecode, bit for bit, and its place in the
serving path (preprocess_input_batch, do_inference_batch, do_inference_coco_batch)."""
import itertools

import numpy as np
import pytest

import jpeg_inputs as JI
import jpeg_oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, jpeg, serve
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import Molder

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (1, 37), (29, 1), (7, 9), (8, 8), (15, 17), (16, 16), (33, 2), (9, 3), (5, 4),
         (517, 771)]


def _molder():
    return Molder(api_utils.get_config())


def _matrix(rng):
    """(name, blob) over sizes x subsamplings x restart settings x qualities x content."""
    out = []
    combos = itertools.product(SIZES, JI.SAMPLINGS, [0, 1, 3, 64])
    for k, ((h, w), samp, rst) in enumerate(combos):
        kind = "noise" if k % 2 else "smooth"
        q = [1, 35, 75, 90, 95, 100][k % 6]
        img = JI.image(rng, h, w, kind, gray=(k % 7 == 0))
        out.append((f"{h}x{w}-{samp}-rst{rst}-q{q}-{kind}",
                    JI.encode(img, q, samp, rst, optimize=(k % 3 == 0))))
    return out


def test_decode_equals_cv2_over_the_matrix_in_mixed_batches(cuda_device):
    rng = np.random.default_rng(0)
    cases = _matrix(rng)
    m = _molder()
    for lo in range(0, len(cases), 37):
        chunk = cases[lo:lo + 37]
        got = m.decode_jpeg_batch([b for _, b in chunk])
        for (name, blob), g in zip(chunk, got):
            ref = JI.cv2_decode(blob)
            assert g.shape == ref.shape, name
            assert np.array_equal(g.cpu().numpy(), ref), name


@pytest.mark.parametrize("q", [1, 50, 90, 100])
def test_decode_equals_cv2_large(cuda_device, q):
    rng = np.random.default_rng(q)
    blobs = [JI.encode(JI.image(rng, 1024, 1024, "noise" if q == 100 else "smooth"), q, "420"),
             JI.encode(JI.image(rng, 2160, 3840), q, "422", rst=5),
             JI.encode(JI.image(rng, 1023, 1025, "noise"), q, "444", optimize=True)]
    got = api_utils.decode_jpeg_batch(blobs)
    for blob, g in zip(blobs, got):
        assert np.array_equal(g.cpu().numpy(), JI.cv2_decode(blob))


def test_coefficients_equal_the_oracle(cuda_device):
    rng = np.random.default_rng(1)
    blobs = [JI.encode(JI.image(rng, 40, 67, "noise"), 95, "420"),
             JI.encode(JI.image(rng, 24, 24), 60, "411", rst=2),
             JI.encode(JI.image(rng, 17, 33, "noise", gray=True), 100, "444"),
             JI.encode(JI.image(rng, 16, 40, "noise"), 80, "440", optimize=True)]
    m = _molder()
    for S in (32, 1024):
        plan = jpeg.Plan(blobs, S)
        d_coef, d_status, _ = m.jpeg_coefficients(plan)
        assert not d_status.cpu().numpy().any()
        got = d_coef.cpu().numpy()
        ref = np.concatenate([jpeg_oracle.coefficients(b)[0] for b in blobs])
        assert np.array_equal(got, ref), S


def test_results_do_not_depend_on_S(cuda_device):
    """S = 32 forces subsequence boundaries inside codewords and many sync rounds."""
    rng = np.random.default_rng(2)
    blobs = [JI.encode(JI.image(rng, 300, 410, "noise"), 97, "420"),
             JI.encode(JI.image(rng, 256, 256), 75, "422", rst=1),
             JI.encode(JI.image(rng, 123, 77), 90, "444", optimize=True)]
    m = _molder()
    ref = [JI.cv2_decode(b) for b in blobs]
    for S in (32, 64, 1024, jpeg.DEFAULT_S, 4096):
        got = m.decode_jpeg_batch(blobs, S=S)
        for g, r in zip(got, ref):
            assert np.array_equal(g.cpu().numpy(), r), S


@pytest.mark.parametrize("big_endian", [False, True])
def test_exif_orientations(cuda_device, big_endian):
    rng = np.random.default_rng(3)
    base = JI.encode(JI.image(rng, 37, 52), 90, "420")
    blobs = [JI.with_exif(base, o, big_endian) for o in range(1, 9)]
    got = api_utils.decode_jpeg_batch(blobs)
    for o, (blob, g) in enumerate(zip(blobs, got), 1):
        ref = JI.cv2_decode(blob)
        assert g.shape == ref.shape and np.array_equal(g.cpu().numpy(), ref), o


def test_spliced_tables_and_colour_spaces(cuda_device):
    rng = np.random.default_rng(4)
    base = JI.encode(JI.image(rng, 45, 61), 85, "420", rst=3)
    blobs = [JI.with_dqt16(base), JI.without_jfif_with_adobe(base, 0),
             JI.without_jfif_with_adobe(base, 1)]
    got = api_utils.decode_jpeg_batch(blobs)
    for blob, g in zip(blobs, got):
        assert np.array_equal(g.cpu().numpy(), JI.cv2_decode(blob))


@pytest.mark.parametrize("corrupt,rst,reason", [
    (JI.truncated, 0, "data ended before the last MCU"),
    (JI.truncated, 2, "RST marker"),
    (JI.with_wrong_rst, 2, "RST marker"),
    (JI.with_bad_code, 0, "bad Huffman code"),
    (JI.with_bad_code, 1, "bad Huffman code"),
    (JI.with_second_scan, 0, "a marker other than EOI"),
])
def test_corrupt_data_raises_after_the_decode(cuda_device, corrupt, rst, reason):
    rng = np.random.default_rng(5)
    good = JI.encode(JI.image(rng, 64, 96, "noise"), 90, "420", rst=rst)
    bad = corrupt(good)
    with pytest.raises(ValueError, match=r"image 1: corrupt JPEG data.*" + reason):
        api_utils.decode_jpeg_batch([good, bad, good])
    # the decoder's buffers are reusable after a refusal
    g, = api_utils.decode_jpeg_batch([good])
    assert np.array_equal(g.cpu().numpy(), JI.cv2_decode(good))


def test_corrupt_restarts_leave_the_other_images_intact(cuda_device):
    """A wrong or missing RSTn leaves unit starts unwritten: with the decoder's scratch filled
    with 0x7F bytes first, the bad images lay out no subsequences and write nothing, and the
    images around them decode as cv2 decodes them."""
    import torch

    rng = np.random.default_rng(9)
    good = JI.encode(JI.image(rng, 64, 96, "noise"), 90, "420", rst=2)
    other = JI.encode(JI.image(rng, 40, 50), 80, "444", rst=1)
    blobs = [other, JI.with_wrong_rst(good), other, JI.truncated(good), other]
    m = _molder()
    plan = jpeg.Plan(blobs)
    m._jpeg_buffer("work", plan.work_words, torch.int32).fill_(0x7F7F7F7F)
    m._jpeg_buffer("unst", plan.unst_bytes, torch.uint8).fill_(0x7F)
    sizes = [h * w * 3 for h, w, _ in plan.shapes]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    out = torch.zeros(int(off[-1]), dtype=torch.uint8, device=m.device)
    st = m.jpeg_decode_into(plan, out, off[:-1]).cpu().numpy()
    assert list(st != 0) == [False, True, False, True, False]
    assert st[1] & N.MRX_JPEG_ST_RST and st[3] & N.MRX_JPEG_ST_RST
    work = m._jpeg_bufs["work"].cpu().numpy()
    ref = JI.cv2_decode(other)
    for b in range(5):
        sub_off, cap = plan.desc[b, jpeg.D_SUB_OFF], plan.desc[b, jpeg.D_SUB_CAP]
        if b in (1, 3):
            assert work[sub_off + 4 * cap] == 0
            assert not out[int(off[b]):int(off[b + 1])].any()
        else:
            got = out[int(off[b]):int(off[b + 1])].view(plan.shapes[b]).cpu().numpy()
            assert np.array_equal(got, ref)


@pytest.mark.parametrize("cut", [4096, 8192])
def test_scan_ending_on_an_unstuff_pass_boundary(cuda_device, cut):
    """The end marker on the first byte of an unstuff pass (16 bytes x 256 threads)."""
    rng = np.random.default_rng(10)
    blob = JI.encode(JI.image(rng, 256, 256, "noise"), 95, "420")
    s = JI.scan_start(blob)
    assert len(blob) - 2 - s > cut
    last = b"\x00" if blob[s + cut - 1] == 0xFF else blob[s + cut - 1:s + cut]
    bad = blob[:s + cut - 1] + last + b"\xff\xd9"
    with pytest.raises(ValueError, match="image 0: corrupt JPEG data.*data ended"):
        api_utils.decode_jpeg_batch([bad, blob])
    got = api_utils.decode_jpeg_batch([blob, blob])
    for g in got:
        assert np.array_equal(g.cpu().numpy(), JI.cv2_decode(blob))


@pytest.mark.parametrize("img_size", [640, None])
def test_preprocess_input_batch_from_bytes_equals_arrays(cuda_device, img_size):
    rng = np.random.default_rng(6)
    if img_size is None:
        blobs = [JI.encode(JI.image(rng, 480, 640), 90, s) for s in ("420", "444", "422")]
    else:
        blobs = [JI.encode(JI.image(rng, 480, 640), 90, "420"),
                 JI.encode(JI.image(rng, 1280, 1280, "noise"), 75, "444", rst=8),
                 JI.encode(JI.image(rng, 97, 333), 95, "422"),
                 JI.encode(JI.image(rng, 640, 640), 60, "420", optimize=True)]
    arrays = [JI.cv2_decode(b) for b in blobs]
    ref = serve.preprocess_input_batch(arrays, img_size)
    got = serve.preprocess_input_batch(blobs, img_size)
    mixed = serve.preprocess_input_batch([blobs[0], arrays[1]] + blobs[2:], img_size)
    for out in (got, mixed):
        assert np.array_equal(out[0], ref[0]) and np.array_equal(out[1], ref[1])
        assert np.array_equal(out[2], ref[2]) and out[3] == ref[3]
    with pytest.raises(TypeError):      # decoded device tensors are not an accepted argument
        serve.preprocess_input_batch(api_utils.decode_jpeg_batch(blobs[:1]), img_size)
    single = serve.preprocess_input(blobs[0], img_size)
    ref_single = serve.preprocess_input(arrays[0], img_size)
    assert np.array_equal(single[0], ref_single[0]) and np.array_equal(single[1], ref_single[1])


def test_do_inference_from_bytes_equals_arrays(cuda_device, tmp_path):
    import random

    import cv2

    from matterport_maskrcnn_with_tensorflow_serving_b200 import visualize
    from test_gpu_anchors_mold import _fake_model

    rng = np.random.default_rng(7)
    blobs = [JI.encode(JI.image(rng, 300, 420), 90, "420"),
             JI.encode(JI.image(rng, 222, 150), 80, "444")]
    arrays = [JI.cv2_decode(b) for b in blobs]
    outs, predict, calls = _fake_model(rng, arrays, 11)
    colors = visualize.random_colors(100, rng=random.Random(6))
    serve.set_predict_fn(predict)
    try:
        calls["k"] = 0
        ref_paths = serve.do_inference_batch(arrays, colors=colors, media_dir=str(tmp_path))
        calls["k"] = 0
        paths = serve.do_inference_batch(blobs, colors=colors, media_dir=str(tmp_path))
        calls["k"] = 0
        ref_coco = serve.do_inference_coco_batch(arrays, [3, 4])
        calls["k"] = 0
        coco = serve.do_inference_coco_batch([blobs[0], arrays[1]], [3, 4])
        calls["k"] = 0
        ref_one = serve.do_inference_unmolded(arrays[0])
        calls["k"] = 0
        one = serve.do_inference_unmolded(blobs[0])
    finally:
        serve.set_predict_fn(None)
    for a, b in zip(ref_paths, paths):
        assert np.array_equal(cv2.imread(a), cv2.imread(b))
    assert coco == ref_coco
    for a, b in zip(ref_one, one):
        assert np.array_equal(a, b)


def test_bench_size_batch(cuda_device):
    """32 files of 1024^2 at quality 90, 4:2:0, no restart markers: one decode."""
    rng = np.random.default_rng(8)
    imgs = [JI.image(rng, 1024, 1024) for _ in range(4)]
    blobs = [JI.encode(imgs[b % 4], 90, "420") for b in range(32)]
    got = api_utils.decode_jpeg_batch(blobs)
    ref = [JI.cv2_decode(blobs[b]) for b in range(4)]
    for b, g in enumerate(got):
        assert np.array_equal(g.cpu().numpy(), ref[b % 4]), b
