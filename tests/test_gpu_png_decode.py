"""The device PNG decoder (csrc/png_decode.cu) against cv2.imdecode, bit for bit, Python's zlib
and a deflate block walker, and its place in the serving path."""
import itertools
import zlib

import numpy as np
import pytest

import jpeg_inputs as JI
import png_decode_inputs as P
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, png, serve
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import Molder
from test_host_png_decode import (after_the_rows_cases, ancillary_cases, corrupt_data_cases,
                                  device_accepts, warning_cases)

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (1, 9), (7, 1), (3, 5), (8, 8), (9, 13), (17, 33)]
STRATEGIES = [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE,
              zlib.Z_FIXED]


def _molder():
    return Molder(api_utils.get_config())


def _check(m, blobs):
    got = m.decode_files(blobs)
    for k, (blob, g) in enumerate(zip(blobs, got)):
        ref = P.cv2_decode(blob)
        assert ref is not None, k
        assert g.shape == ref.shape and np.array_equal(g.cpu().numpy(), ref), k


def _matrix(rng):
    out = []
    for k, ((ct, depth), (h, w), il) in enumerate(itertools.product(P.COMBOS, SIZES, (0, 1))):
        kind = ("noise", "smooth", "constant")[k % 3]
        filters = [(0, 1, 2, 3, 4), (4,), (3,), (1,), (2,), (0,)][k % 6]
        pal = P.default_palette(max(1, (1 << depth) - (k % 3))) if ct == 3 else None
        a = P.samples(rng, h, w, ct, depth, kind)
        out.append(P.write(a, ct, depth, interlace=il, filters=filters, level=[0, 1, 6, 9][k % 4],
                           strategy=STRATEGIES[k % 5], palette=pal))
    return out


def test_decode_equals_cv2_over_the_matrix_in_mixed_batches(cuda_device):
    rng = np.random.default_rng(0)
    blobs = _matrix(rng)
    jpegs = [JI.encode(JI.image(rng, 23, 31), 90, "420"), JI.encode(JI.image(rng, 8, 8), 75)]
    m = _molder()
    for lo in range(0, len(blobs), 41):
        _check(m, blobs[lo:lo + 41] + jpegs)
    _check(m, [blob for _, blob, _ in ancillary_cases()])


def test_zlib_settings(cuda_device):
    rng = np.random.default_rng(1)
    a = P.samples(rng, 37, 45, 2, 8, "smooth")
    b = P.samples(rng, 37, 45, 6, 8, "noise")
    blobs = []
    for k, (level, strategy) in enumerate(itertools.product((0, 1, 6, 9), STRATEGIES)):
        for wbits in range(9, 16):                     # every window, every memLevel
            img, ct = (a, 2) if k % 2 else (b, 6)
            blobs.append(P.write(img, ct, 8, level=level, strategy=strategy, wbits=wbits,
                                 mem=1 + (k + wbits) % 9))
    for wbits, mem in itertools.product(range(9, 16), range(1, 10)):
        blobs.append(P.write(a, 2, 8, level=6, wbits=wbits, mem=mem))
    m = _molder()
    for lo in range(0, len(blobs), 60):
        _check(m, blobs[lo:lo + 60])


def test_cv2_and_own_encoder_files(cuda_device):
    import cv2

    rng = np.random.default_rng(2)
    img = JI.image(rng, 61, 83)
    blobs = []
    for level in range(10):
        for strategy in (cv2.IMWRITE_PNG_STRATEGY_DEFAULT, cv2.IMWRITE_PNG_STRATEGY_FILTERED,
                         cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY, cv2.IMWRITE_PNG_STRATEGY_RLE,
                         cv2.IMWRITE_PNG_STRATEGY_FIXED):
            ok, buf = cv2.imencode(".png", img[..., ::-1], [cv2.IMWRITE_PNG_COMPRESSION, level,
                                                            cv2.IMWRITE_PNG_STRATEGY, strategy])
            blobs.append(buf.tobytes())
    _check(_molder(), blobs)
    imgs = [JI.image(rng, 40, 57), JI.image(rng, 1, 1), JI.image(rng, 129, 3)]
    back = api_utils.decode_png_batch(api_utils.encode_png_batch(imgs))
    for x, y in zip(imgs, back):
        assert np.array_equal(x, y.cpu().numpy())


def test_adam7_split_and_exif(cuda_device):
    rng = np.random.default_rng(3)
    blobs = []
    for o in range(1, 9):
        a = P.samples(rng, 6 + o, 11, 2, 8)
        where = "before" if o % 2 else "after"
        blobs.append(P.write(a, 2, 8, interlace=o % 2, **{where: [P.exif_chunk(o, o > 4)]}))
    blobs.append(P.write(P.samples(rng, 30, 20, 6, 16), 6, 16, split=1, interlace=1))
    blobs.append(P.write(P.samples(rng, 5, 70, 0, 1), 0, 1, split=7))
    _check(_molder(), blobs)


@pytest.mark.parametrize("h,w,ct,depth", [(1024, 1024, 2, 8), (2160, 3840, 2, 8),
                                          (1024, 1024, 6, 16)])
def test_large(cuda_device, h, w, ct, depth):
    import cv2

    rng = np.random.default_rng(h + depth)
    rgb = JI.image(rng, h, w)
    if ct == 2:
        blob = cv2.imencode(".png", rgb[..., ::-1])[1].tobytes()
    else:
        a = np.concatenate([rgb.astype(np.uint16) * 257 + 3, np.full((h, w, 1), 9, np.uint16)], -1)
        blob = P.write(a, 6, 16, filters=(4, 1, 2, 3))
    _check(_molder(), [blob, blob])


def test_inflated_stream_and_block_list(cuda_device):
    rng = np.random.default_rng(4)
    blobs = [P.write(P.samples(rng, h, w, 2, 8, kind), 2, 8, filters=(0,), level=lv,
                     strategy=st, mem=mem)
             for h, w, kind, lv, st, mem in [
                 (40, 33, "noise", 6, 0, 1), (40, 33, "smooth", 9, 0, 1),
                 (400, 400, "constant", 1, zlib.Z_RLE, 1), (40, 33, "noise", 0, 0, 8),
                 (40, 33, "smooth", 6, zlib.Z_FIXED, 2)]]
    m = _molder()
    plan = png.DecodePlan(blobs)
    sizes = [h * w * 3 for h, w, _ in plan.shapes]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    import torch
    out = torch.empty(int(off[-1]), dtype=torch.uint8, device="cuda")
    d_status, d_info, d_blocks = m.png_decode_into(plan, out, off[:-1])
    assert not d_status.cpu().numpy().any()
    filt = m._jpeg_buffer("png_filt", plan.filt_bytes, torch.uint8).cpu().numpy()
    info, blocks = d_info.cpu().numpy(), d_blocks.cpu().numpy()
    for b, blob in enumerate(blobs):
        z = P.zlib_stream(blob)
        D = plan.desc[b]
        n = int(D[png.DD_N])
        got = filt[int(D[png.DD_FILT_OFF]):int(D[png.DD_FILT_OFF]) + n]
        assert got.tobytes() == zlib.decompressobj().decompress(z)      # filter 0: unchanged
        true = P.deflate_blocks(z)
        assert info[b, 0] == len(true) and info[b, 2] == n
        assert len(true) <= D[png.DD_BLK_CAP]
        mine = blocks[int(D[png.DD_BLK_OFF]):int(D[png.DD_BLK_OFF]) + len(true)]
        # bits count from the zlib stream's first byte: the deflate stream starts at bit 16
        assert [tuple(r) for r in mine] == [(16 + s, o) for s, o, _, _ in true], b
    # one colour: copies that reach back into earlier blocks, block after block
    assert info[2, 0] > 3


def test_corrupt_data_raises_and_buffers_are_reusable(cuda_device):
    m = _molder()
    good = P.write(P.samples(np.random.default_rng(5), 20, 17, 2, 8), 2, 8)
    after = [(name, P.with_zlib_stream(good, z), ok) for name, z, ok in after_the_rows_cases()]
    refused = corrupt_data_cases() + [(n, b) for n, b, ok in after if not device_accepts(ok)]
    for name, blob in refused:
        with pytest.raises(ValueError, match="image 1: corrupt PNG data"):
            m.decode_files([good, blob, good])
    for name, blob in warning_cases() + [(n, b) for n, b, ok in after if device_accepts(ok)]:
        _check(m, [good, blob])


def test_every_block_measured_in_the_chain_gives_the_same_images(cuda_device):
    """With no candidate slots the chain measures every block itself; the images are the same,
    and with slots the chain takes (almost) every block from the finder."""
    import cv2

    rng = np.random.default_rng(10)
    blobs = [cv2.imencode(".png", JI.image(rng, 300, 400)[..., ::-1])[1].tobytes(),
             P.write(P.samples(rng, 200, 150, 6, 16, "smooth"), 6, 16, level=9, mem=1),
             P.write(P.samples(rng, 90, 70, 3, 4, "smooth"), 3, 4, interlace=1, level=6, mem=2),
             P.write(P.samples(rng, 64, 64, 2, 8, "smooth"), 2, 8, level=6,
                     strategy=zlib.Z_FIXED)]
    m = _molder()
    ref = [g.cpu().numpy() for g in m.decode_png_batch(blobs, slots=0)]
    for slots in (0, 1, 4, 32):
        got = m.decode_png_batch(blobs, slots=slots)
        for k, (g, r, blob) in enumerate(zip(got, ref, blobs)):
            assert np.array_equal(g.cpu().numpy(), r), (slots, k)
            assert np.array_equal(r, P.cv2_decode(blob)), k
    import torch
    for slots in (0, 4):
        plan = png.DecodePlan(blobs, slots=slots)
        sizes = [h * w * 3 for h, w, _ in plan.shapes]
        out = torch.empty(sum(sizes), dtype=torch.uint8, device="cuda")
        _, d_info, _ = m.png_decode_into(plan, out, np.cumsum([0] + sizes)[:-1])
        info = d_info.cpu().numpy()
        for b, blob in enumerate(blobs):
            true = P.deflate_blocks(P.zlib_stream(blob))
            dynamic = sum(t == 2 for _, _, t, _ in true)
            assert info[b, 0] == len(true), (slots, b)
            if slots == 0:
                assert info[b, 1] == len(true) and info[b, 6] == 0, b
            else:         # the finder finds every dynamic block; stored and fixed ones are measured
                assert info[b, 1] == len(true) - dynamic and info[b, 6] >= dynamic, b


def test_references_across_many_blocks(cuda_device):
    """One colour at memLevel 1: hundreds of short blocks whose copies reach back across block
    after block, resolved in order; and an image with more blocks than its list holds."""
    import cv2

    one = np.full((512, 512, 3), 77, np.uint8)
    one[::97, ::89] = 3
    blobs = [P.write(one, 2, 8, filters=(0,), level=9, mem=1),
             P.write(one, 2, 8, filters=(1,), level=1, strategy=zlib.Z_RLE, mem=1),
             cv2.imencode(".png", one[..., ::-1])[1].tobytes()]
    _check(_molder(), blobs)
    assert len(P.deflate_blocks(P.zlib_stream(blobs[0]))) > 20
    tiny = P.write(P.samples(np.random.default_rng(11), 2, 40, 2, 8), 2, 8, level=0, mem=1,
                   strategy=zlib.Z_HUFFMAN_ONLY)
    z = P.zlib_stream(tiny)
    # many empty stored blocks ahead of the data: more blocks than the list holds
    raw = zlib.decompress(z)
    empties = b"\x00\x00\x00\xff\xff" * (png.block_capacity(len(raw), 5 * 300) + 5)
    stored = b"\x78\x01" + empties + b"\x01" + len(raw).to_bytes(2, "little") + \
        (0xFFFF ^ len(raw)).to_bytes(2, "little") + raw + zlib.adler32(raw).to_bytes(4, "big")
    many = P.with_zlib_stream(tiny, stored)
    hd = png.parse(many)
    assert len(P.deflate_blocks(P.zlib_stream(many))) > png.block_capacity(hd.filtered,
                                                                            hd.zlib_len)
    _check(_molder(), [many, blobs[0]])


def test_serve_entry_points_with_png_jpeg_and_arrays(cuda_device, tmp_path):
    import random

    import cv2

    from matterport_maskrcnn_with_tensorflow_serving_b200 import visualize
    from test_gpu_anchors_mold import _fake_model

    rng = np.random.default_rng(7)
    blobs = [cv2.imencode(".png", JI.image(rng, 300, 420)[..., ::-1])[1].tobytes(),
             JI.encode(JI.image(rng, 222, 150), 80, "444"),
             P.write(P.samples(rng, 97, 130, 3, 4), 3, 4, interlace=1,
                     after=[P.exif_chunk(6)])]
    arrays = [P.cv2_decode(b) for b in blobs]
    for size in (640, None):
        same = blobs[:1] * 2 if size is None else blobs
        ref_arrays = arrays[:1] * 2 if size is None else arrays
        ref = serve.preprocess_input_batch(ref_arrays, size)
        got = serve.preprocess_input_batch(same, size)
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    single = serve.preprocess_input(blobs[2])
    assert np.array_equal(single[0], serve.preprocess_input(arrays[2])[0])
    with pytest.raises(ValueError, match="image 1: neither a JPEG nor a PNG file"):
        serve.preprocess_input_batch([blobs[0], b"GIF89a...."])
    outs, predict, calls = _fake_model(rng, arrays, 11)
    colors = visualize.random_colors(100, rng=random.Random(6))
    serve.set_predict_fn(predict)
    try:
        calls["k"] = 0
        ref_paths = serve.do_inference_batch(arrays, colors=colors, media_dir=str(tmp_path))
        calls["k"] = 0
        paths = serve.do_inference_batch(blobs, colors=colors, media_dir=str(tmp_path))
        calls["k"] = 0
        ref_coco = serve.do_inference_coco_batch(arrays, [3, 4, 5])
        calls["k"] = 0
        coco = serve.do_inference_coco_batch([blobs[0], arrays[1], blobs[2]], [3, 4, 5])
        calls["k"] = 0
        ref_one = serve.do_inference(arrays[0], colors=colors, media_dir=str(tmp_path))
        calls["k"] = 0
        one = serve.do_inference(blobs[0], colors=colors, media_dir=str(tmp_path))
    finally:
        serve.set_predict_fn(None)
    for a, b in zip(ref_paths + [ref_one], paths + [one]):
        assert np.array_equal(cv2.imread(a), cv2.imread(b))
    assert coco == ref_coco


def test_bench_size_batch(cuda_device):
    """32 files of 1024^2 as cv2.imwrite writes them: one decode."""
    import cv2

    rng = np.random.default_rng(8)
    imgs = [JI.image(rng, 1024, 1024) for _ in range(4)]
    blobs = [cv2.imencode(".png", imgs[b % 4][..., ::-1])[1].tobytes() for b in range(32)]
    got = api_utils.decode_png_batch(blobs)
    for b, g in enumerate(got):
        assert np.array_equal(g.cpu().numpy(), imgs[b % 4]), b
