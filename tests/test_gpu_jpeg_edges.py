"""The device JPEG decoder (csrc/jpeg.cu) on tests/jpeg_edge_inputs.py's files, read from the
committed tests/golden/jpeg_edges.npz: IDCT arithmetic past the range encoders write, 16-bit
quantisers, colour and upsampling extremes, DC prediction sums, entropy-code corners, and their
progressive re-encodings.  Pixels are held to the golden cv2.imdecode output and to the oracle,
coefficients to the oracle, refusals to the image index; through api_utils.decode_jpeg_batch and
Molder.decode_jpeg_batch at S = 32, 1024 and 4096, in mixed batches of baseline and progressive
files.  The golden file, not the GPU host's cv2, is the reference: its libjpeg-turbo may run other
SIMD code."""
import functools
import hashlib
import os

import numpy as np
import pytest

import jpeg_edge_inputs as E
import jpeg_oracle as O
import jpeg_progressive_oracle as PO
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, jpeg
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import Molder

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_edges.npz")


@functools.lru_cache(maxsize=None)
def golden():
    g = np.load(GOLDEN)
    return {k: g[k] for k in g.files}


def _cases():
    """(name, blob, expected) of every file; expected is the golden decode (an array, or
    (shape, sha256)), or None where cv2 refuses the file."""
    g = golden()
    files, off = g["files"].tobytes(), g["file_off"]
    out = []
    for i, name in enumerate(g["names"]):
        name = str(name)
        blob = files[off[i]:off[i + 1]]
        if not g["cv2_ok"][i]:
            exp = None
        elif "px_" + name in g:
            exp = g["px_" + name]
        else:
            exp = (tuple(int(v) for v in g["shape"][i]), str(g["px_sha256"][i]))
        out.append((name, blob, exp))
    return out


def _progressive(blob):
    return jpeg._frame_marker(blob) == 0xC2


# the files the device refuses: every one cv2 refuses, and a DC sum past int32 that cv2's
# libjpeg-turbo lets wrap when it comes before the last ~512 bytes (DESIGN §3.20)
REFUSED = {"dc_symbol_16": "bogus Huffman table", "dc_int32_overflow": "overflows int32"}


def _accepted():
    return [c for c in _cases() if c[0] not in REFUSED]


def _check(name, img, exp):
    img = img.cpu().numpy()
    if isinstance(exp, tuple):
        assert img.shape == exp[0] and hashlib.sha256(img.tobytes()).hexdigest() == exp[1], name
    else:
        assert img.shape == exp.shape, name
        diff = int((img != exp).any(axis=-1).sum())
        assert diff == 0, f"{name}: {diff} pixels differ from cv2"


def _mixed_batches(cases, n=23):
    """Batches of up to n files, baseline and progressive interleaved."""
    base = [c for c in cases if not _progressive(c[1])]
    prog = [c for c in cases if _progressive(c[1])]
    order = [c for pair in zip(base, prog) for c in pair]
    order += base[len(prog):] + prog[len(base):]
    return [order[i:i + n] for i in range(0, len(order), n)]


def test_golden_names_cover_the_refusals():
    names = {c[0] for c in _cases()}
    assert set(REFUSED) <= names
    assert {n for n, _, e in _cases() if e is None} == {"dc_symbol_16"}


def test_api_utils_decode_equals_golden_cv2(cuda_device):
    for batch in _mixed_batches(_accepted()):
        got = api_utils.decode_jpeg_batch([b for _, b, _ in batch])
        for (name, _, exp), img in zip(batch, got):
            _check(name, img, exp)


@pytest.mark.parametrize("S", [32, 1024, 4096])
def test_molder_decode_equals_golden_and_oracle(cuda_device, S):
    m = Molder(api_utils.get_config())
    for batch in _mixed_batches(_accepted(), n=31):
        got = m.decode_jpeg_batch([b for _, b, _ in batch], S=S)
        for (name, blob, exp), img in zip(batch, got):
            _check(name, img, exp)
            if S == 1024:
                ref = (PO if _progressive(blob) else O).decode(blob)
                assert np.array_equal(img.cpu().numpy(), ref), name


def test_coefficients_equal_the_oracle(cuda_device):
    m = Molder(api_utils.get_config())
    acc = _accepted()
    base = [b for _, b, _ in acc if not _progressive(b)]
    prog = [b for _, b, _ in acc if _progressive(b)]
    for S in (32, 4096):
        d_coef, d_status, _ = m.jpeg_coefficients(jpeg.Plan(base, S))
        assert not d_status.cpu().numpy().any(), S
        ref = np.concatenate([O.coefficients(b)[0] for b in base])
        assert np.array_equal(d_coef.cpu().numpy(), ref), S
    d_coef, d_status, _ = m.jpeg_progressive_coefficients(jpeg.ProgressivePlan(prog))
    assert not d_status.cpu().numpy().any()
    ref = np.concatenate([PO.coefficients(b)[0] for b in prog])
    assert np.array_equal(d_coef.cpu().numpy(), ref)


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refusals_name_the_image(cuda_device, name):
    cases = {c[0]: c for c in _cases()}
    bad = cases[name][1]
    good = [c for c in _accepted() if c[0].startswith("idct_random")][:2]
    prog = [c for c in _accepted() if _progressive(c[1])][:1]
    blobs = [good[0][1], prog[0][1], bad, good[1][1]]
    with pytest.raises(ValueError, match=r"image 2: .*" + REFUSED[name]):
        api_utils.decode_jpeg_batch(blobs)
    # the decoder's buffers are reusable after a refusal
    got = api_utils.decode_jpeg_batch([blobs[0], blobs[1], blobs[3]])
    for (n, _, exp), img in zip([good[0], prog[0], good[1]], got):
        _check(n, img, exp)


def test_full_colour_grids(cuda_device):
    """Every (Y, Cr), (Y, Cb) and (Cb, Cr) pair of DC-only 4:4:4 blocks, 2048 x 2048 each."""
    g = golden()
    grids = E.colour_grids(step=1)
    got = api_utils.decode_jpeg_batch([c.blob for c in grids])
    for c, img in zip(grids, got):
        assert hashlib.sha256(img.cpu().numpy().tobytes()).hexdigest() == \
            str(g["grid_sha256_" + c.name]), c.name
