"""Every mask-expand kernel computes the sample csrc/expand.cuh defines, bit for bit.

The float64 parity tests (test_gpu_unmold.py and the others using helpers.check_values) hold the
kernels within 1e-6 of upstream and excuse a mask pixel whose float64 value lies within 1e-6 of
0.5.  That band hides the one-ulp departures a kernel could make (> for >=, a split FMA, rem / D
for rem * (1/D), a reciprocal rounded the wrong way, vertical-first interpolation) and every
threshold tie.  Here there is no band: each kernel's output is compared with
expand_oracle's restatement of the float32 definition,

  - mrx_mask_expand_values (team kernel shapes): every in-box value bitwise, NaN equal to NaN;
  - mrx_mask_expand: the whole byte canvas, zero outside every box;
  - mrx_mask_expand_packed: the packed planes, padding bits included;
  - mrx_rle_count / mrx_rle_write: the run lengths of every instance,

on the input families and kernel paths of expand_inputs.py: tiles at threshold ties, near 0.5 by
a few ulps, dyadic, at the extents where the floor estimate is corrected, float64 values that
round onto 0.5, subnormals and signed zeros, and non-finite values (which must set nothing
outside a box), plus two smooth synthetic images of the benchmark's shape."""
import numpy as np
import pytest

from helpers import pad_rows, prepared_engine

import expand_inputs as ei
import expand_oracle as eo

pytestmark = pytest.mark.gpu


def _mismatch(path, what, b, bad, got, want, planes=False):
    """Assertion message: how many elements differ, the first as (b, k, y, x), both values and
    the path.  bad marks the differing elements of got / want ([H, W, N], or [N, H, WB] packed
    planes, whose x is then a byte)."""
    where = np.argwhere(bad)
    idx = tuple(int(v) for v in where[0])
    k, y, x = idx if planes else (idx[2], idx[0], idx[1])
    return (f"{path}: {what} differs at {len(where)} elements; first (b, k, y, x) = "
            f"({b}, {k}, {y}, {x}): got {got[idx]!r}, want {want[idx]!r}")


def _same_values(got, want):
    """bitwise equal, NaN equal to NaN"""
    return (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))


def check_kernels(path, ims, R, dtype, mask_hw, boxes=None, classes=ei.CLASSES):
    """Run every expand kernel that takes the shape on `ims` (R detection rows each, mask tiles
    of `dtype`) and compare each output with the restatement.  boxes: the intended boxes of each
    image, checked against the device's."""
    import torch

    eng = prepared_engine(ims, R, classes, dtype, mask_hw)
    counts, d_boxes, cls, _ = eng.fetch_meta()
    counts, d_boxes, cls = counts.copy(), d_boxes.copy(), cls.copy()
    src = eng.d_src_index.cpu().numpy()
    want = []
    for b, im in enumerate(ims):
        k = int(counts[b])
        if boxes is not None:
            assert np.array_equal(d_boxes[b, :k], boxes[b]), f"{path}: image {b} boxes"
        tiles = im.mrcnn_mask[src[b, :k], :, :, cls[b, :k]]
        want.append(eo.expand(im.original_image_shape[:2], d_boxes[b, :k], tiles))
    lane = eng.mw <= ei.LANE_MASK_W

    def canvas(b):
        return eng.canvas_view(b, int(counts[b])).cpu().numpy().view(np.bool_)

    if lane:
        # the team kernel's values (NaN-filled: outside the boxes nothing may be stored)
        d_values = torch.full((int(eng._offsets[len(ims)]),), float("nan"), dtype=torch.float32,
                              device="cuda")
        try:
            eng.enqueue_expand_values(d_values)
        except Exception as e:      # R past the team kernel's limit: no values to compare
            assert "status -2" in str(e), e
            d_values = None
        for b, (m, v) in enumerate(want if d_values is not None else []):
            H, W, k = m.shape
            o = int(eng._offsets[b])
            got_v = d_values[o:o + H * W * k].view(H, W, k).cpu().numpy()
            ok = _same_values(got_v, v)
            assert ok.all(), _mismatch(path, "values (team kernel)", b, ~ok, got_v, v)
            c = canvas(b)
            assert np.array_equal(c, m), _mismatch(path, "canvas of the values launch", b,
                                                   c != m, c, m)
    eng.d_canvas.fill_(7)                 # every byte of the result must be rewritten
    eng.enqueue_expand()
    for b, (m, _) in enumerate(want):
        c = eng.canvas_view(b, int(counts[b])).cpu().numpy()
        assert np.array_equal(c, m.view(np.uint8)), _mismatch(path, "byte canvas", b,
                                                              c != m.view(np.uint8), c, m)
    if not lane:
        return
    eng._packed_buffer()
    eng.d_packed.fill_(0xAA)              # every packed byte must be rewritten
    d_packed, off = eng.enqueue_expand_packed()
    for b, (m, _) in enumerate(want):
        H, W, k = m.shape
        wb = (W + 7) // 8
        got = d_packed[int(off[b]):int(off[b]) + k * H * wb].cpu().numpy().reshape(k, H, wb)
        exp = eo.packed(m)
        assert np.array_equal(got, exp), _mismatch(path, "packed planes", b, got != exp, got,
                                                   exp, planes=True)
    d_runs, off = eng.enqueue_rle()
    runs = d_runs.cpu().numpy().view(np.uint32)
    for b, (m, _) in enumerate(want):
        for n, exp in enumerate(eo.rle_runs(m)):
            i = b * R + n
            got = runs[int(off[i]) + i:int(off[i + 1]) + i + 1]
            assert np.array_equal(got, exp), (
                f"{path}: RLE of (b, k) = ({b}, {n}) differs: {len(got)} runs, want {len(exp)}; "
                f"first differing run {int(np.argmax(got[:len(exp)] != exp[:len(got)]))}")


CASES = [(f, p) for f in ei.FAMILIES for p in ei.PATHS]


@pytest.mark.parametrize("family,path", CASES, ids=[f"{f}-{p}" for f, p in CASES])
def test_kernels_equal_the_definition(cuda_device, family, path):
    im, R, dtype, boxes = ei.case(family, path)
    check_kernels(f"{family}/{path}", [im], R, dtype, ei.PATHS[path][1], [boxes])


def test_kernels_equal_the_definition_two_images(cuda_device):
    """Two images of different shapes in one launch: the per-image tables and slots."""
    a, R, dtype, ba = ei.case("near", "team_aligned", 1)
    b, _, _, bb = ei.case("near", "team_unaligned", 2)
    check_kernels("near/two_images", [a, pad_rows(b, R)], R, dtype, (28, 28), [ba, bb])


def test_nonfinite_sets_nothing_outside_the_box(cuda_device):
    """Tiles of +inf alone: every sample inside a box is inf or NaN, and the lanes of columns
    outside a box interpolate the same values through the shuffles.  Nothing outside a box may be
    set, in the canvas, the planes (their padding bits) or the runs."""
    rng = np.random.default_rng(77)
    H, W, n = 120, 333, 12
    boxes = ei._boxes(rng, (H, W), rng.integers(1, 100, n), rng.integers(1, 120, n), False)
    tiles = np.full((n, 28, 28), np.inf)
    tiles[::3] = -np.inf
    tiles[1::3, ::2] = np.nan
    im = ei.make_image((H, W), boxes, tiles, n)
    check_kernels("inf/outside_box", [im], n, np.float64, (28, 28), [boxes])


@pytest.mark.parametrize("which", ["configs1", "bench0"])
def test_synth_images_equal_the_definition(cuda_device, which):
    """Smooth synthetic tiles at the benchmark's scale: a BASELINE.json configs[1] image (1024 x
    1024, 100 instances, molded) and the first image of bench.py's batch."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import synth

    if which == "configs1":
        im = synth.make_batch(93, 1, (1024, 1024), 100)[0]
    else:
        import bench
        im = bench.make_bench_images(0, 1)[0]
    check_kernels(which, [im], im.detections.shape[0], np.float32, (28, 28),
                  classes=im.mrcnn_mask.shape[-1])
