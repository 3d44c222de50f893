"""CPU tests of the COCO restatements in coco_oracle.py: compressed RLE strings against answers
worked out by hand from the published format, the string round trip, and the results builder."""
import numpy as np
import pytest

import oracle
from coco_oracle import build_coco_results, encode, rle_from_string, rle_to_string


# Worked by hand: x is split into 5-bit groups from the least significant end; a group is
# followed by another (0x20 added) until the rest is the sign extension of the group's bit 0x10.
@pytest.mark.parametrize("counts,want", [
    ([5], b"5"),
    ([0, 16], b"0`0"),                  # 16 = 0b10000: bit 0x10 set, so a 0 group follows
    ([3, 2, 1, 4], b"3212"),            # run 3: 4 - 2 = 2
    ([10, 5, 3, 1], b":53L"),           # run 3: 1 - 5 = -4 -> group 28, '0' + 28 = 'L'
    ([8294400], b"PPTm7"),              # an empty 2160x3840 mask: 5 groups
    ([1, 2147483646, 1], b"1nooooo11"),  # 2^31 - 2 takes 7 characters
])
def test_known_strings(counts, want):
    assert rle_to_string(counts) == want
    assert rle_from_string(want) == counts


@pytest.mark.parametrize("counts", [
    [], [0], [7], [0, 1], [3, 4], [0, 5, 9], [2, 2, 2], [1, 1, 1, 1], [0, 1, 2, 3, 4],
    [31, 32, 15, 16, 17, 1 << 20, 1, (1 << 31) - 1, 0, 5],
])
def test_round_trip_edge_cases(counts):
    assert rle_from_string(rle_to_string(counts)) == counts


def test_round_trip_random_runs():
    rng = np.random.default_rng(5)
    for _ in range(300):
        n = int(rng.integers(1, 40))
        scale = int(rng.choice([2, 40, 3000, 1 << 22]))
        counts = [int(v) for v in rng.integers(0, scale, size=n)]
        s = rle_to_string(counts)
        assert rle_from_string(s) == counts
        assert all(48 <= c < 48 + 64 for c in s)


def test_encode_of_masks():
    """encode() is rle_encode + rle_to_string: an empty mask, a set first pixel (leading 0 run),
    and a random mask that decodes back."""
    assert encode(np.zeros((3, 4), bool)) == {"size": [3, 4], "counts": b"<"}    # one run of 12
    m = np.zeros((2, 2), bool)
    m[0, 0] = True
    assert encode(m)["counts"] == rle_to_string([0, 1, 3]) == b"013"
    r = np.random.default_rng(6).random((17, 23)) < 0.4
    rle = encode(np.asfortranarray(r))
    back = oracle.rle_decode({"size": rle["size"], "counts": rle_from_string(rle["counts"])})
    assert np.array_equal(back, r)


def test_build_coco_results_fields():
    H, W = 6, 5
    rois = np.array([[1, 0, 4, 3], [0, 2, 6, 5]], np.int32)
    class_ids = np.array([3, 1], np.int32)
    scores = np.array([0.875, 0.5], np.float32)
    masks = np.zeros((H, W, 2), bool)
    masks[1:4, 0:3, 0] = True
    masks[:, 2:5, 1] = True
    cat = [0, 11, 12, 13]
    res = build_coco_results([42], rois, class_ids, scores, masks, category_ids=cat)
    assert len(res) == 2
    r0, r1 = res
    assert r0["image_id"] == 42 and r0["category_id"] == 13 and r1["category_id"] == 11
    assert r0["bbox"] == [0, 1, 3, 3] and r1["bbox"] == [2, 0, 3, 6]
    assert r0["score"] == np.float32(0.875) and r1["score"] == np.float32(0.5)
    # column-major: columns 0-2 hold rows 1-3 set, i.e. 1 zero, 3 ones, 3 zeros, ... 16 zeros
    assert r0["segmentation"] == {"size": [H, W], "counts": rle_to_string([1, 3, 3, 3, 3, 3, 14])}
    assert r1["segmentation"]["counts"] == rle_to_string([12, 18])
    # identity categories; upstream repeats the detections for every image id it is given
    res = build_coco_results([1, 2], rois, class_ids, scores, masks)
    assert [r["image_id"] for r in res] == [1, 1, 2, 2]
    assert [r["category_id"] for r in res] == [3, 1, 3, 1]
    assert build_coco_results([1], None, None, None, None) == []
