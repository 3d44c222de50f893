"""The device JPEG encoder (csrc/jpeg_encode.cu) against cv2.imencode('.jpg') byte for byte over
the input matrix at every quality and both optimize settings, its coefficients and bit counts
against jpeg_encode_oracle, and its place in the serving path (do_inference[_batch] with
image_format="jpeg", display_instances(save_path="x.jpg"))."""
import random

import numpy as np
import pytest
import torch

import jpeg_encode_inputs as I
import jpeg_encode_oracle as O
import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, serve, synth, visualize
from matterport_maskrcnn_with_tensorflow_serving_b200 import jpeg_encode as je

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

MATRIX = I.matrix()
SMALL = [n for n, img in MATRIX if img.shape[0] * img.shape[1] <= 480 * 640]


def cv2_jpeg(img, quality=95, optimize=False):
    return cv2.imencode(".jpg", np.ascontiguousarray(img[..., ::-1]),
                        [cv2.IMWRITE_JPEG_QUALITY, int(quality),
                         cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize)])[1].tobytes()


@pytest.mark.parametrize("optimize", I.OPTIMIZE)
@pytest.mark.parametrize("quality", I.QUALITIES)
def test_encode_jpeg_batch_equals_cv2(cuda_device, quality, optimize):
    """The whole matrix in one mixed-size batch, from tensors."""
    names = [n for n, _ in MATRIX]
    arrays = [img for _, img in MATRIX]
    files = api_utils.encode_jpeg_batch([torch.from_numpy(a).to(cuda_device) for a in arrays],
                                        quality, optimize)
    assert len(files) == len(names)
    for name, a, got in zip(names, arrays, files):
        assert got == cv2_jpeg(a, quality, optimize), name


@pytest.mark.parametrize("optimize", I.OPTIMIZE)
def test_encode_jpeg_batch_from_arrays_at_the_default_quality(cuda_device, optimize):
    imgs = dict(MATRIX)
    arrays = [imgs[n] for n in SMALL]
    files = api_utils.encode_jpeg_batch(arrays, optimize=optimize)
    for name, a, got in zip(SMALL, arrays, files):
        assert got == cv2_jpeg(a, 95, optimize), name


@pytest.mark.parametrize("quality,optimize", [(95, False), (100, True), (10, False)])
def test_device_intermediates_equal_the_oracle(cuda_device, quality, optimize):
    """Every block's quantised coefficients (dummy blocks included), and per image the coded
    bits, bytes, stuffed zeros, header and file lengths."""
    imgs = dict(MATRIX)
    files, info, coef, plan = api_utils._jpeg_encode([imgs[n] for n in SMALL], quality,
                                                     optimize, stats=True)
    for b, name in enumerate(SMALL):
        data, e = O.encode(imgs[name], quality, optimize)
        assert files[b] == data, name
        k0 = int(plan.desc[b, je.D_BLK_OFF])
        assert np.array_equal(coef[k0:k0 + e.coef.shape[0]], e.coef), name
        row = info[b]
        assert row[N.MRX_JPEG_ENC_BITS] == e.bits, name
        assert row[N.MRX_JPEG_ENC_BYTES] == e.bytes, name
        assert row[N.MRX_JPEG_ENC_FF] == e.ff, name
        assert row[N.MRX_JPEG_ENC_HDR] == e.hdr, name
        assert row[N.MRX_JPEG_ENC_FILE] == len(data), name
        assert row[N.MRX_JPEG_ENC_BLOCKS] == e.coef.shape[0], name
        assert len(data) <= je.file_bound(e.coef.shape[0])


def test_noise_at_quality_100_within_the_bound(cuda_device):
    rng = np.random.default_rng(5)
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in
            [(256, 256), (333, 517), (1, 1)]] + [I.checkerboard(130, 77)]
    files, info, _, plan = api_utils._jpeg_encode(imgs, 100, stats=True)
    for b, img in enumerate(imgs):
        assert files[b] == cv2_jpeg(img, 100)
        assert len(files[b]) <= je.file_bound(int(plan.desc[b, je.D_NBLK]))
        assert info[b, N.MRX_JPEG_ENC_FF] > 0 or img.shape[0] == 1


def test_decode_of_encoded_equals_cv2_imdecode(cuda_device):
    imgs = dict(MATRIX)
    names = ["overlay250x371", "noise37x53", "const1x40", "checker4_33x47", "synth120x161"]
    files = api_utils.encode_jpeg_batch([imgs[n] for n in names], 90)
    decoded = api_utils.decode_jpeg_batch(files)
    for name, blob, got in zip(names, files, decoded):
        ref = cv2.cvtColor(cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR),
                           cv2.COLOR_BGR2RGB)
        assert np.array_equal(got.cpu().numpy(), ref), name


def test_refusal_before_launch(cuda_device):
    with pytest.raises(ValueError, match="image 1"):
        api_utils.encode_jpeg_batch([np.zeros((2, 2, 3), np.uint8), np.zeros((2, 2, 4), np.uint8)])
    with pytest.raises(ValueError, match="quality"):
        api_utils.encode_jpeg_batch([np.zeros((2, 2, 3), np.uint8)], quality=-5)
    assert api_utils.encode_jpeg_batch([]) == []


def test_do_inference_writes_cv2_bytes(cuda_device, tmp_path):
    """image_format="jpeg": do_inference and do_inference_batch write .jpg files with the bytes
    cv2.imencode('.jpg') gives for the oracle's overlay; the default still writes the PNG."""
    from test_gpu_anchors_mold import _fake_model

    rng = np.random.default_rng(51)
    imgs = [synth.synth_rgb_image(rng, 300, 420), synth.synth_rgb_image(rng, 222, 150)]
    outs, predict, calls = _fake_model(rng, imgs, 17)
    colors = visualize.random_colors(100, rng=random.Random(9))
    overlays = []
    for img, (im, molded, meta, window) in zip(imgs, outs):
        rb, rc, rs, rm = oracle.unmold_detections(
            im.detections.astype(np.float64), im.mrcnn_mask.astype(np.float64), img.shape,
            molded.shape, window)
        overlays.append(oracle.composite_instances(img, rb, rm, colors))
    serve.set_predict_fn(predict)
    try:
        calls["k"] = 0
        one = serve.do_inference(imgs[0], colors=colors, media_dir=str(tmp_path),
                                 image_format="jpeg")
        calls["k"] = 0
        paths = serve.do_inference_batch(imgs, colors=colors, media_dir=str(tmp_path),
                                         image_format="jpeg", quality=80)
        calls["k"] = 0
        default = serve.do_inference(imgs[0], colors=colors, media_dir=str(tmp_path))
    finally:
        serve.set_predict_fn(None)
    assert one.endswith(".jpg") and all(p.endswith(".jpg") for p in paths)
    with open(one, "rb") as f:
        assert f.read() == cv2_jpeg(overlays[0])
    for path, ov in zip(paths, overlays):
        with open(path, "rb") as f:
            assert f.read() == cv2_jpeg(ov, 80)
    assert default.endswith(".png")
    with open(default, "rb") as f:
        assert f.read() == cv2.imencode(".png", np.ascontiguousarray(overlays[0][..., ::-1]))[1] \
            .tobytes()


def test_do_inference_refuses_a_bad_format(cuda_device):
    with pytest.raises(ValueError, match="image_format"):
        api_utils._unmold_overlay_file_batch([], [], image_format="gif")


@pytest.mark.parametrize("ext", [".jpg", ".JPEG"])
def test_display_instances_save_path(cuda_device, tmp_path, ext):
    rng = np.random.default_rng(53)
    h, w, n = 200, 261, 4
    image = synth.synth_rgb_image(rng, h, w)
    boxes = np.array([[10, 20, 90, 120], [50, 60, 180, 250], [0, 0, 0, 0], [100, 5, 199, 80]],
                     np.int32)
    masks = np.zeros((h, w, n), bool)
    for i, (y1, x1, y2, x2) in enumerate(boxes):
        masks[y1:y2, x1:x2, i] = rng.random((y2 - y1, x2 - x1)) < 0.7
    colors = visualize.random_colors(n, rng=random.Random(4))
    path = str(tmp_path / f"out{ext}")
    out = visualize.display_instances(image, boxes, masks, colors=colors, save_path=path)
    ref = oracle.composite_instances(image, boxes, masks, colors)
    assert np.array_equal(out, ref)
    cv2.imwrite(str(tmp_path / "ref.jpg"), ref[:, :, ::-1])
    with open(path, "rb") as f, open(tmp_path / "ref.jpg", "rb") as g:
        assert f.read() == g.read()
