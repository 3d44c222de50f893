"""The device PNG encoder (csrc/png.cu) against cv2.imencode('.png') byte for byte, its
intermediates against png_oracle, and its place in the serving path (do_inference[_batch],
display_instances(save_path=))."""
import random

import numpy as np
import pytest
import torch

import oracle
import png_inputs
import png_oracle as P
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, serve, synth, visualize

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

MATRIX = png_inputs.matrix()


def _cv2_png(img):
    return cv2.imencode(".png", np.ascontiguousarray(img[..., ::-1]))[1].tobytes()


def _batches():
    """The matrix in mixed-size batches of up to 7 images."""
    names = [name for name, _ in MATRIX]
    return [names[i:i + 7] for i in range(0, len(names), 7)]


@pytest.mark.parametrize("source", ["tensor", "array"])
@pytest.mark.parametrize("batch", range(len(_batches())))
def test_encode_png_batch_equals_cv2(cuda_device, batch, source):
    imgs = dict(MATRIX)
    names = _batches()[batch]
    arrays = [imgs[n] for n in names]
    inputs = [torch.from_numpy(a).to(cuda_device) for a in arrays] if source == "tensor" else arrays
    files = api_utils.encode_png_batch(inputs)
    assert len(files) == len(names)
    for name, a, got in zip(names, arrays, files):
        assert got == _cv2_png(a), name


def test_device_intermediates_equal_the_oracle(cuda_device):
    """Symbol counts, block types and block bit lengths, image by image."""
    names = ["sym16383", "runs", "noise300x200", "synth240x320", "overlay480x640", "noise333x1",
             "const1x7"]
    imgs = dict(MATRIX)
    files, img_info, blk_info, plan = api_utils._png_encode([imgs[n] for n in names], stats=True)
    from matterport_maskrcnn_with_tensorflow_serving_b200 import png

    for b, name in enumerate(names):
        data, e = P.encode(imgs[name])
        assert files[b] == data, name
        assert img_info[b, N.MRX_PNG_IMG_NSYM] == e.nsym, name
        assert img_info[b, N.MRX_PNG_IMG_NBLK] == len(e.blocks), name
        assert img_info[b, N.MRX_PNG_IMG_FILE] == len(data), name
        k0 = int(plan.desc[b, png.D_BLK_OFF])
        rows = blk_info[k0:k0 + len(e.blocks)]
        assert list(rows[:, N.MRX_PNG_BLK_TYPE]) == [blk.type for blk in e.blocks], name
        assert list(rows[:, N.MRX_PNG_BLK_BITS]) == [blk.bits for blk in e.blocks], name
        assert list(rows[:, N.MRX_PNG_BLK_BIT]) == [blk.bit_start for blk in e.blocks], name


def test_refusal_before_launch(cuda_device):
    with pytest.raises(ValueError, match="image 1"):
        api_utils.encode_png_batch([np.zeros((2, 2, 3), np.uint8), np.zeros((2, 2), np.uint8)])
    assert api_utils.encode_png_batch([]) == []


def test_do_inference_writes_cv2_bytes(cuda_device, tmp_path):
    """do_inference and do_inference_batch write the bytes cv2.imwrite writes for the oracle's
    overlay (oracle.composite_instances of the oracle's unmold)."""
    from test_gpu_anchors_mold import _fake_model

    rng = np.random.default_rng(41)
    imgs = [synth.synth_rgb_image(rng, 300, 420), synth.synth_rgb_image(rng, 222, 150)]
    outs, predict, calls = _fake_model(rng, imgs, 17)
    colors = visualize.random_colors(100, rng=random.Random(8))
    refs = []
    for img, (im, molded, meta, window) in zip(imgs, outs):
        rb, rc, rs, rm = oracle.unmold_detections(
            im.detections.astype(np.float64), im.mrcnn_mask.astype(np.float64), img.shape,
            molded.shape, window)
        refs.append(_cv2_png(oracle.composite_instances(img, rb, rm, colors)))
    serve.set_predict_fn(predict)
    try:
        calls["k"] = 0
        one = serve.do_inference(imgs[0], colors=colors, media_dir=str(tmp_path))
        calls["k"] = 0
        paths = serve.do_inference_batch(imgs, colors=colors, media_dir=str(tmp_path))
    finally:
        serve.set_predict_fn(None)
    with open(one, "rb") as f:
        assert f.read() == refs[0]
    for path, ref in zip(paths, refs):
        with open(path, "rb") as f:
            assert f.read() == ref


def test_do_inference_write_failure_raises_ioerror(cuda_device, tmp_path):
    from test_gpu_anchors_mold import _fake_model

    rng = np.random.default_rng(43)
    img = synth.synth_rgb_image(rng, 120, 90)
    _, predict, _ = _fake_model(rng, [img], 5)
    blocker = tmp_path / "file"
    blocker.write_bytes(b"")
    serve.set_predict_fn(predict)
    try:
        with pytest.raises(IOError):
            serve.do_inference(img, media_dir=str(blocker / "sub"))
    finally:
        serve.set_predict_fn(None)


def test_display_instances_save_path(cuda_device, tmp_path):
    rng = np.random.default_rng(47)
    h, w, n = 200, 260, 4
    image = synth.synth_rgb_image(rng, h, w)
    boxes = np.array([[10, 20, 90, 120], [50, 60, 180, 250], [0, 0, 0, 0], [100, 5, 199, 80]],
                     np.int32)
    masks = np.zeros((h, w, n), bool)
    for i, (y1, x1, y2, x2) in enumerate(boxes):
        masks[y1:y2, x1:x2, i] = rng.random((y2 - y1, x2 - x1)) < 0.7
    colors = visualize.random_colors(n, rng=random.Random(3))
    path = str(tmp_path / "out.png")
    out = visualize.display_instances(image, boxes, masks, colors=colors, save_path=path)
    ref = oracle.composite_instances(image, boxes, masks, colors)
    assert np.array_equal(out, ref)
    with open(path, "rb") as f:
        assert f.read() == _cv2_png(ref)
