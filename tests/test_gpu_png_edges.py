"""The device PNG decoder (csrc/png_decode.cu) on the edge inputs of tests/png_edge_inputs.py:
pixels equal to cv2.imdecode bit for bit through both entry points in batches mixed with JPEG
files, refusals by image index with the expected MRX_PNG_ST_* bit, the same images at 0, 1, 4 and
32 candidate slots, and the chain's block, measure and candidate counts against the walker and
the restated finder."""
import functools

import numpy as np
import pytest

import jpeg_inputs as JI
import png_decode_inputs as P
import png_edge_inputs as E
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, png
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import Molder

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _cases():
    return E.all_cases()


def _valid():
    return [c for c in _cases() if c.pixels is not None]


def _jpegs():
    rng = np.random.default_rng(3)
    return [JI.encode(JI.image(rng, 23, 31), 90, "420"), JI.encode(JI.image(rng, 8, 8), 75)]


def _assert_pixels(got, cases):
    for g, c in zip(got, cases):
        g = g.cpu().numpy() if hasattr(g, "cpu") else g
        assert g.shape == c.pixels.shape and np.array_equal(g, c.pixels), c.name
        assert np.array_equal(P.cv2_decode(c.blob), c.pixels), c.name


def test_decode_files_mixed_with_jpeg(cuda_device):
    m = Molder(api_utils.get_config())
    cases, jpegs = _valid(), _jpegs()
    blobs = []
    for k, c in enumerate(cases):
        blobs += [c.blob, jpegs[k % 2]]
    got = m.decode_files(blobs)
    _assert_pixels(got[0::2], cases)
    # the deflate edges again with the stream in 7-byte IDAT chunks (1-byte for small streams)
    small = [c for c in cases if c.raw is not None and len(c.blob) < 100000]
    split = [P.with_zlib_stream(c.blob, P.zlib_stream(c.blob), 1 if len(c.blob) < 3000 else 7)
             for c in small]
    _assert_pixels(m.decode_files(split + jpegs)[:len(small)], small)


def test_api_utils_decode_png_batch(cuda_device):
    cases = _valid()
    _assert_pixels(api_utils.decode_png_batch([c.blob for c in cases]), cases)


def _run(m, blobs, slots):
    import torch

    plan = png.DecodePlan(blobs, slots=slots)
    sizes = [h * w * 3 for h, w, _ in plan.shapes]
    off = np.cumsum([0] + sizes)
    out = torch.zeros(int(off[-1]), dtype=torch.uint8, device="cuda")
    d_status, d_info, _ = m.png_decode_into(plan, out, off[:-1])
    out = out.cpu().numpy()
    imgs = [out[off[b]:off[b + 1]].reshape(plan.shapes[b]) for b in range(plan.B)]
    return d_status.cpu().numpy(), d_info.cpu().numpy(), imgs


def test_refusals_name_the_image_and_set_the_status(cuda_device):
    m = Molder(api_utils.get_config())
    good = _valid()[0]
    jpeg = _jpegs()[0]
    refused = [c for c in _cases() if c.pixels is None]
    for c in refused:
        z = P.zlib_stream(c.blob)
        for split in (None, 1, 7):
            blob = P.with_zlib_stream(c.blob, z, split)
            with pytest.raises(ValueError, match="image 1: corrupt PNG data"):
                m.decode_files([jpeg, blob, good.blob])
    blobs = [good.blob] + [c.blob for c in refused]
    for slots in (0, 4):
        st, _, imgs = _run(m, blobs, slots)
        assert st[0] == 0 and np.array_equal(imgs[0], good.pixels)
        for c, s in zip(refused, st[1:]):
            assert s == c.status, (c.name, slots, s)


def _expected_seq(z, blocks, cand, K):
    """(fewest, most) blocks the chain measures itself at K slots: stored, fixed and
    reach-before-start blocks always; a dynamic block in a tile with more candidates than K
    slots maybe (which candidates win the slots is a race)."""
    per = {}
    for x in cand:
        per[x // E.TILE_BITS] = per.get(x // E.TILE_BITS, 0) + 1
    lo = hi = 0
    for b in blocks:
        if b["type"] != 2 or K == 0 or b["need"] > b["out"]:
            lo += 1
            hi += 1
        elif per.get(b["bit"] // E.TILE_BITS, 0) > K:
            hi += 1
    return lo, hi


def test_slots_give_the_same_images_and_the_chain_counts(cuda_device):
    m = Molder(api_utils.get_config())
    cases = [c for c in _cases() if c.raw is not None or c.pixels is None]
    blobs = [c.blob for c in cases]
    walks = [E.walk(P.zlib_stream(b)) for b in blobs]
    cands = [E.candidates(P.zlib_stream(b)) if len(b) < 20000 else None for b in blobs]
    ref = None
    exact = 0
    for slots in (0, 1, 4, 32):
        st, info, imgs = _run(m, blobs, slots)
        for k, (c, s, img) in enumerate(zip(cases, st, imgs)):
            _, blocks = walks[k]
            if c.pixels is None:
                assert s == c.status, (c.name, slots)
                continue
            assert s == 0 and np.array_equal(img, c.pixels), (c.name, slots)
            assert info[k, 0] == len(blocks), (c.name, slots)           # MRX_PNG_DEC_NBLK
            assert info[k, 2] == len(c.raw), (c.name, slots)            # MRX_PNG_DEC_OUT
            if cands[k] is None:
                continue
            z = P.zlib_stream(c.blob)
            if slots:
                assert info[k, 6] == len(cands[k]), (c.name, slots)     # MRX_PNG_DEC_CAND
                ndyn = sum(b["type"] == 2 for b in blocks)
                if c.counts.get("false_candidates") or c.counts.get("false_to_end"):
                    assert info[k, 6] > ndyn, c.name
            lo, hi = _expected_seq(z, blocks, cands[k], slots)
            assert lo <= info[k, 1] <= hi, (c.name, slots, info[k, 1], lo, hi)   # MRX_PNG_DEC_SEQ
            exact += lo == hi
        if ref is None:
            ref = imgs
        for c, a, b in zip(cases, ref, imgs):
            if c.pixels is not None:
                assert np.array_equal(a, b), (c.name, slots)
    assert exact > 40
    # the dense file overfills 1 and 4 slots: the chain measures some of its dynamic blocks
    dense = next(k for k, c in enumerate(cases) if c.name == "one literal per dynamic block")
    _, info, _ = _run(m, [blobs[dense]], 1)
    assert info[0, 1] > 0
