"""The output layout of a planned batch (engine.BatchLayout), on the host without a device: slot
offsets against an independent restatement of both rounding rules, the configs[3] layout whose
offsets pass 2^32, each geometry the plan refuses at its boundary, and the kept-instance walk."""
import re

import numpy as np
import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200.engine import BatchLayout, make_geom


def _geom(H, W):
    return make_geom((H, W, 3), (H, W, 3), (0, 0, H, W))


def _restated_offsets(shapes, R):
    """Byte canvas: H*W*R per image rounded up to 256.  Packed: R*H*ceil(W/8) rounded up to 16."""
    canvas, packed = [0], [0]
    for H, W in shapes:
        canvas.append(canvas[-1] + -(-(H * W * R) // 256) * 256)
        packed.append(packed[-1] + -(-(R * H * -(-W // 8)) // 16) * 16)
    return canvas, packed


@pytest.mark.parametrize("shapes,R", [
    ([(799, 1333), (333, 517), (2, 2), (1023, 1024), (97, 1333)], 100),   # W = 1333, W % 8 != 0
    ([(799, 1333), (5, 9), (2, 3), (1024, 1024)], 1),
    ([(3, 1333), (600, 1001)], 3),
])
def test_offsets_equal_the_restated_rules(shapes, R):
    lay = BatchLayout([_geom(H, W) for H, W in shapes], R)
    canvas, packed = _restated_offsets(shapes, R)
    # the batches exercise both roundings
    assert any((b - a) != H * W * R for (a, b), (H, W) in zip(zip(canvas, canvas[1:]), shapes))
    assert any((b - a) != R * H * -(-W // 8)
               for (a, b), (H, W) in zip(zip(packed, packed[1:]), shapes))
    assert lay.canvas_off.dtype == np.int64 and lay.packed_off.dtype == np.int64
    assert lay.canvas_off.tolist() == canvas and lay.packed_off.tolist() == packed
    assert (lay.n, lay.R) == (len(shapes), R)
    assert lay.geom.dtype == np.int32 and lay.geom.shape == (len(shapes), 8)
    assert (lay.max_h, lay.max_w) == (max(H for H, _ in shapes), max(W for _, W in shapes))
    for b, (H, W) in enumerate(shapes):
        assert lay.hw(b) == (H, W)
        for k in (0, 1, R):
            assert lay.canvas_span(b, k) == (canvas[b], canvas[b] + H * W * k)
            assert lay.packed_shape(b, k) == (k, H, -(-W // 8))
            assert lay.packed_span(b, k) == (packed[b], packed[b] + k * H * -(-W // 8))
        assert lay.canvas_span(b, R)[1] <= canvas[b + 1]
        assert lay.packed_span(b, R)[1] <= packed[b + 1]
    counts = np.arange(len(shapes), dtype=np.int32) % (R + 1)
    assert lay.canvas_bytes(counts) == sum(H * W * int(k) for (H, W), k in zip(shapes, counts))


def test_configs3_layout_passes_2_to_the_32():
    """BASELINE configs[3]: 12 images of 2160x3840 at R = 50, as one GPU's share is planned."""
    B, H, W, R = 12, 2160, 3840, 50
    slot, pslot = 414_720_000, 51_840_000
    assert slot == H * W * R and pslot == R * H * (W // 8)
    lay = BatchLayout([_geom(H, W)] * B, R)
    assert lay.canvas_off.tolist() == [b * slot for b in range(B + 1)]
    assert lay.packed_off.tolist() == [b * pslot for b in range(B + 1)]
    assert int(lay.canvas_off[B - 1]) > 1 << 32 and int(lay.canvas_off[B]) > 1 << 32
    for b in range(B):
        assert lay.canvas_span(b, 0) == (b * slot, b * slot)
        assert lay.canvas_span(b, R) == (b * slot, (b + 1) * slot)
        assert lay.packed_span(b, 0) == (b * pslot, b * pslot)
        assert lay.packed_span(b, R) == (b * pslot, (b + 1) * pslot)


_PIXELS = "canvas larger than 2^30 pixels is not supported"
_BYTES = "a canvas of H*W*R >= 2^31 bytes is not supported (32-bit chunk math)"
_SIDES = "image sides must be >= 2"


@pytest.mark.parametrize("R,refused,accepted,message", [
    # 2^30 + 1 pixels is refused, 2^15 x 2^15 = 2^30 is taken
    (1, (5, 214748365), (1 << 15, 1 << 15), _PIXELS),
    # H*W*R = 2^31 - 2^20 is refused; 13919 * 51403 * 3 = 2^31 - 2^20 - 1 is taken
    (2, (1 << 15, 32752), (13919, 51403), _BYTES),
])
def test_each_size_limit_at_its_boundary(R, refused, accepted, message):
    H, W = refused
    assert (H * W == (1 << 30) + 1) if message == _PIXELS else (H * W * R == (1 << 31) - (1 << 20))
    with pytest.raises(ValueError, match=re.escape(message)):
        BatchLayout([_geom(2, 2), _geom(H, W)], R)
    R_ok = R if message == _PIXELS else 3
    H, W = accepted
    assert H * W <= 1 << 30 and H * W * R_ok < (1 << 31) - (1 << 20)
    lay = BatchLayout([_geom(H, W)], R_ok)
    assert int(lay.canvas_off[1]) == -(-(H * W * R_ok) // 256) * 256


@pytest.mark.parametrize("side", range(4))
def test_a_side_of_one_is_refused(side):
    g = _geom(64, 48)
    g[side] = 1
    with pytest.raises(ValueError, match=re.escape(_SIDES)):
        BatchLayout([_geom(8, 8), g], 5)
    g[side] = 2
    BatchLayout([_geom(8, 8), g], 5)


def test_without_limits_a_one_pixel_high_mask_has_a_layout():
    """visualize stages caller-held masks this way; their kernels take sides of 1."""
    lay = BatchLayout([[1, 37, 1, 37, 0, 0, 1, 37]], 3, limits=False)
    assert lay.canvas_off.tolist() == [0, 256] and lay.canvas_span(0, 3) == (0, 111)
    assert lay.packed_off.tolist() == [0, 16] and lay.packed_span(0, 3) == (0, 15)


def test_kept_instances_skip_empty_images():
    lay = BatchLayout([_geom(4, 4)] * 6, 4)
    counts = np.array([2, 0, 3, 0, 0, 1], np.int32)
    assert list(lay.kept_instances(counts)) == [
        (0, 0, 0), (0, 1, 1), (2, 0, 8), (2, 1, 9), (2, 2, 10), (5, 0, 20)]
    assert list(lay.kept_instances([0] * 6)) == []
    assert list(lay.kept_instances([4] * 6)) == [
        (b, k, 4 * b + k) for b in range(6) for k in range(4)]
