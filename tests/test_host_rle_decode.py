"""COCO RLE ground truth on the host side: the string format's known answers, the packing of a
batch's strings and runs (engine.pack_rle), every ValueError raised before an upload, and the
argument checks of mrx_rle_parse and mrx_rle_decode."""
import ctypes as C

import numpy as np
import pytest

import coco_oracle as co
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import MaskBatch, pack_rle

# worked by hand from the published format (pycocotools maskApi.c rleToString / rleFrString)
KNOWN = [
    ([0, 4], b"04"),
    ([5, 2, 1, 3], b"5211"),
    ([2, 5, 2, 1], b"252L"),       # cnts[3] - cnts[1] = -4: a negative delta
    ([100], b"T3"),
    ([16], b"`0"),                 # 16 needs two groups: its bit 0x10 would read as the sign
]


# (what is wrong, null argument, B, R) of "Output slots"; every row is MRX_E_INVALID
BAD_SLOTS = [
    ("null slot base", "base", 1, 100),
    ("null offsets", "off", 1, 100),
    ("null counts", "counts", 1, 100),
    ("null geom", "geom", 1, 100),
    ("B > MRX_MAX_BATCH", None, N.MRX_MAX_BATCH + 1, 100),
    ("R = 0", None, 0, 0),
    ("R = 65535", None, 0, 65535),
]


def _geom(H, W):
    return [H, W, H, W, 0, 0, H, W]


@pytest.mark.parametrize("counts,string", KNOWN)
def test_known_strings(counts, string):
    assert co.rle_to_string(counts) == string
    assert co.rle_from_string(string) == counts


def test_pack_mixed_kinds():
    """bytes, str and count lists of two images pack into one string buffer and one runs array;
    instance i = b*R + k, R the larger image's count."""
    rles = [[{"size": [2, 2], "counts": b"04"}, {"size": [2, 2], "counts": [1, 2, 1]},
             {"size": [2, 2], "counts": "T3"}],
            [{"size": [3, 4], "counts": np.array([12], np.uint32)},
             {"size": [3, 4], "counts": b"5211"}]]
    pk = pack_rle([_geom(2, 2), _geom(3, 4)], [[1, 2, 3], [4, 5]], rles)
    assert pk["R"] == 3 and pk["counts"].tolist() == [3, 2]
    assert pk["strings"].tobytes() == b"04T35211"
    assert pk["str_off"].tolist() == [0, 2, 2, 4, 4, 8, 8]
    assert pk["runs"].dtype == np.uint32 and pk["runs"].tolist() == [1, 2, 1, 12]
    S = 8
    assert pk["run_off"].tolist() == [0, S + 0, 2, S + 3, 4, 8]
    assert pk["run_count"].tolist() == [0, 3, 0, 1, 0, 0]


def test_pack_empty_batch_parts():
    pk = pack_rle([_geom(4, 4), _geom(5, 5)], [[], []], [[], []])
    assert pk["R"] == 1 and pk["strings"].size == 0 and pk["runs"].size == 0
    assert pk["str_off"].tolist() == [0, 0, 0]


@pytest.mark.parametrize("rles,cls,match", [
    ([[{"size": [4, 5], "counts": b"0"}]], [[1]], r"image 0, instance 0: size \[4, 5\] is not"),
    ([[{"size": [4, 4], "counts": b"0"}, {"size": [4, 4], "counts": 16}]], [[1, 1]],
     "image 0, instance 1: counts must be"),
    ([[{"size": [4, 4], "counts": [1.0, 15.0]}]], [[1]], "image 0, instance 0: counts must be"),
    ([[{"size": [4, 4], "counts": [[16]]}]], [[1]], "image 0, instance 0: counts must be"),
    ([[{"size": [4, 4], "counts": [0, 16]}], [{"size": [4, 4], "counts": [17, -1]}]], [[1], [1]],
     "image 1, instance 0: an uncompressed count is negative"),
    ([[{"size": [4, 4], "counts": [2 ** 32, 0]}]], [[1]],
     "image 0, instance 0: an uncompressed count is negative or does not fit"),
    ([[{"size": [4, 4], "counts": "0é"}]], [[1]], "image 0, instance 0: .*not ASCII"),
    ([[{"size": [4, 4]}]], [[1]], "image 0, instance 0: an RLE is a dict"),
    ([[{"size": [4, 4], "counts": b"`0"}]], [[1, 2]], r"image 0: \(2,\) class ids for 1 RLE"),
    ([[{"size": [4, 4], "counts": b"`0"}]], [[2 ** 40]], "image 0: class ids must be integers"),
])
def test_host_errors_before_upload(rles, cls, match):
    """Each bad input raises ValueError naming the image (and the instance) before anything is
    uploaded: no library or device is needed to get there."""
    with pytest.raises(ValueError, match=match):
        MaskBatch.from_rle(None, None, [_geom(4, 4)] * len(rles), cls, rles)


def test_image_count_mismatch():
    with pytest.raises(ValueError, match="1 RLE lists and 2 class-id arrays for 2 images"):
        pack_rle([_geom(4, 4)] * 2, [[], []], [[]])


def _parse(lib, s, off, cnt, runs, rc, st, B, R):
    return lib.mrx_rle_parse(s, off, cnt, runs, rc, st, B, R, None)


def test_parse_argument_checks():
    lib = N.load()
    p = C.c_void_p(16)
    for null in range(6):
        args = [None if j == null else p for j in range(6)]
        assert _parse(lib, *args, 1, 10) == -1, null
        assert lib.mrx_last_error().decode().startswith("mrx_rle_parse:")
    for B, R in [(N.MRX_MAX_BATCH + 1, 10), (-1, 10), (0, 0), (0, 65535)]:
        assert _parse(lib, p, p, p, p, p, p, B, R) == -1, (B, R)
        assert lib.mrx_last_error().decode().startswith("mrx_rle_parse:")
    assert _parse(lib, p, p, p, p, p, p, 0, 10) == 0


def _decode(lib, base, off, cnt, geom, B, R, runs=16, run_off=16, run_count=16, ends=16,
            status=16, max_h=16, max_w=16):
    v = lambda x: None if x is None else C.c_void_p(x)   # noqa: E731
    return lib.mrx_rle_decode(v(runs), v(run_off), v(run_count), v(ends), v(status), cnt, geom,
                              off, base, B, R, max_h, max_w, None)


def test_decode_slot_checks():
    """mrx_rle_decode checks the output slots as every other packed-slot entry point does (the
    same bad slots as the slot test of the other entry points), then its pointers and extents."""
    lib = N.load()
    for what, null, B, R in BAD_SLOTS:
        args = {k: (None if k == null else C.c_void_p(16)) for k in ("base", "off", "counts", "geom")}
        assert _decode(lib, args["base"], args["off"], args["counts"], args["geom"], B, R) == -1, what
        assert lib.mrx_last_error().decode().startswith("mrx_rle_decode:"), what
    p = C.c_void_p(16)
    for name in ("runs", "run_off", "run_count", "ends", "status"):
        assert _decode(lib, p, p, p, p, 1, 10, **{name: None}) == -1, name
        assert lib.mrx_last_error().decode().startswith("mrx_rle_decode:")
    for h, w in [(0, 16), (16, 0)]:
        assert _decode(lib, p, p, p, p, 1, 10, max_h=h, max_w=w) == -1
        assert lib.mrx_last_error().decode().startswith("mrx_rle_decode:")
    assert _decode(lib, p, p, p, p, 0, 10) == 0
