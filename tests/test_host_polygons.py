"""COCO polygon ground truth on the host side: the layout engine.pack_polygons gives
mrx_poly_decode, every ValueError MaskBatch.from_coco raises before an upload, the argument
checks of mrx_poly_decode, and COCOevalSegm's default refusal of polygons."""
import ctypes as C

import numpy as np
import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import evaluate
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import MaskBatch, pack_polygons


def _geom(H, W):
    return [H, W, H, W, 0, 0, H, W]


def test_pack_layout():
    """Two images, instance i = b*R + k: polygons (one of two parts, one with an odd number),
    a box list and an RLE dict that is left to pack_rle."""
    segms = [[[[0, 0, 10, 0, 10, 10], [1.5, 2, 3, 4, 5, 6, 7]],
              {"size": [20, 30], "counts": b"0"},
              [[1, 2, 3, 4]]],
             [[[-0.15, 0.1, 4, 4, 0, 4]]]]
    pk = pack_polygons([_geom(20, 30), _geom(8, 9)], [[1, 2, 3], [4]], segms)
    assert pk["R"] == 3 and pk["counts"].tolist() == [3, 1] and pk["P"] == 4
    assert pk["poly"].tolist() == [True, False, True, True, False, False]
    assert pk["rle"].tolist() == [False, True, False, False, False, False]
    assert pk["vert"].dtype == np.int32
    # (int)(5 * c + .5): 1.5 -> 8, -0.15 -> 0 (truncation, not floor), 0.1 -> 1
    assert pk["vert"].tolist() == [[0, 0], [50, 0], [50, 50],
                                   [8, 10], [15, 20], [25, 30],
                                   [5, 10], [5, 30], [20, 30], [20, 10],   # box 1,2 4x4
                                   [0, 1], [20, 20], [0, 20]]
    assert pk["part_vert"].tolist() == [0, 3, 6, 10, 13]
    assert pk["part_inst"].tolist() == [0, 0, 2, 3]
    assert pk["inst_part"].tolist() == [0, 2, 2, 3, 4, 4, 4]
    assert pk["part_col"].tolist() == [0, 31, 62, 93, 103]
    # per edge min(W, (|dx| + 2) // 5 + 1) + 1
    assert pk["part_tog"].tolist()[:2] == [0, (11 + 1) + (1 + 1) + (11 + 1)]
    assert np.diff(pk["part_tog"]).min() > 0


@pytest.mark.parametrize("segms,match", [
    ([[[]]], "image 0, instance 0: an empty polygon list"),
    ([[[[1, 2, 3]]]], "image 0, instance 0: the first part has 3 numbers"),
    ([[[[1, 2, 3, 4], [1, 2, 3, 4, 5, 6]]]], "image 0, instance 0: a box list .* not 4 numbers"),
    ([[[[1, 2, 3, 4, 5, 6], [7]]]], "image 0, instance 0: part 1 has 1 numbers"),
    ([[[[1, 2, 3, 4, 5, 6], []]]], "image 0, instance 0: part 1 has 0 numbers"),
    ([[[[1, 2, 3, 4, 5, np.nan]]]], "image 0, instance 0: a coordinate is NaN or infinite"),
    ([[[[1, 2, 3, 4, 5, np.inf]]]], "image 0, instance 0: a coordinate is NaN or infinite"),
    ([[[[1, 2, "x", 4, 5, 6]]]], "image 0, instance 0: part 0 is not a list of numbers"),
    ([[[[1, 2, [3], 4, 5, 6]]]], "image 0, instance 0: part 0 is not"),
    ([[[[1, 2, 3, 4, 5e8, 6]]]], "image 0, instance 0: a coordinate scaled by 5 does not fit"),
    ([[[[-3e8, 2, 3, 4, 3e8, 6]]]], "image 0, instance 0: two consecutive vertices"),
    ([[[[1, 2, 3, 4, 5, 6]], "abc"]], "image 0, instance 1: a segmentation is a polygon list"),
    ([[[[1, 2, 3, 4, 5, 6]], {"size": [9, 9], "counts": b"0"}]],
     r"image 0, instance 1: size \[9, 9\] is not"),
])
def test_host_errors_before_upload(segms, match):
    """Each bad input raises ValueError naming the image and the instance before anything is
    uploaded: no library or device is needed to get there."""
    cls = [np.ones(len(s), np.int32) for s in segms]
    with pytest.raises(ValueError, match=match):
        MaskBatch.from_coco(None, None, [_geom(4, 4)] * len(segms), cls, segms)


def test_count_mismatches():
    with pytest.raises(ValueError, match=r"image 0: \(2,\) class ids for 1 segmentations"):
        MaskBatch.from_coco(None, None, [_geom(4, 4)], [[1, 2]], [[[[0, 0, 1, 1, 2, 0]]]])
    with pytest.raises(ValueError, match="1 segmentation lists and 2 class-id arrays for 2"):
        pack_polygons([_geom(4, 4)] * 2, [[], []], [[]])


def test_from_rle_still_refuses_polygons():
    with pytest.raises(ValueError, match="image 0, instance 0: an RLE is a dict"):
        MaskBatch.from_rle(None, None, [_geom(4, 4)], [[1]], [[[[0, 0, 1, 1, 2, 0]]]])


def test_cocoeval_refuses_polygons_by_default():
    ann = {"category_id": 1, "segmentation": [[0, 0, 1, 1, 2, 0]], "area": 1.0}
    with pytest.raises(ValueError, match="polygon segmentations are not supported"):
        evaluate.COCOevalSegm().add_results([], [[ann]], [1])
    with pytest.raises(ValueError, match="2 image shapes for 1 images"):
        evaluate.COCOevalSegm(polygons=True).add_results([], [[ann]], [1], [(4, 6), (4, 6)])


def _poly(lib, B=1, R=10, P=1, max_h=16, max_w=16, **null):
    names = ["vert", "part_vert", "part_inst", "part_col", "part_tog", "inst_part", "tog",
             "col_start", "carry", "counts", "geom", "off", "base"]
    p = {k: (None if k in null else C.c_void_p(16)) for k in names}
    return lib.mrx_poly_decode(p["vert"], p["part_vert"], p["part_inst"], p["part_col"],
                               p["part_tog"], P, p["inst_part"], p["tog"], p["col_start"],
                               p["carry"], p["counts"], p["geom"], p["off"], p["base"], B, R,
                               max_h, max_w, None)


def test_poly_decode_argument_checks():
    """"Output slots" first (null slot pointers, B and R), then the other pointers, P and the
    extents; every message names mrx_poly_decode.  B = 0 or P = 0 launches nothing."""
    lib = N.load()

    def bad(**kw):
        assert _poly(lib, **kw) == -1, kw
        assert lib.mrx_last_error().decode().startswith("mrx_poly_decode:"), kw

    for name in ("base", "off", "counts", "geom", "vert", "part_vert", "part_inst", "part_col",
                 "part_tog", "inst_part", "tog", "col_start", "carry"):
        bad(**{name: True})
    for B, R in [(N.MRX_MAX_BATCH + 1, 10), (-1, 10), (1, 0), (1, 65535)]:
        bad(B=B, R=R)
    bad(P=-1)
    bad(max_h=0)
    bad(max_w=0)
    assert _poly(lib, B=0) == 0
    assert _poly(lib, P=0) == 0
