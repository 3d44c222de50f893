"""The contour tracer (csrc/contours.cu) on the inputs of tests/contour_edge_inputs.py: saddles on
word and chunk seams, regions that cut the planes, cycle lengths around the pointer-jumping round
counts, totals around the scan tiles, and coordinates past 2^23.  Every polygon must equal
`contour_oracle.mask_polygons` of the mask zeroed outside its clamped region, exactly and in
order, through `engine.trace_packed_contours` (hand-built regions on np.packbits planes) and
through the NumPy entry's trace (`visualize.mask_contours`); every raw output must also keep the
trace's invariants."""
import numpy as np
import pytest

import contour_edge_inputs as E
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import visualize
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import (BatchLayout, _download_contours,
                                                                     contours_to_lists,
                                                                     trace_packed_contours)

pytestmark = pytest.mark.gpu

GB = 1e9


def _assert_same(got, want, what):
    assert len(got) == len(want), f"{what}: {len(got)} contours, want {len(want)}"
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.dtype == np.float64 and g.shape == w.shape, f"{what}: contour {i} {g.shape} {w.shape}"
        if not np.array_equal(g, w):
            j = int(np.flatnonzero((g != w).any(axis=1))[0])
            raise AssertionError(f"{what}: contour {i} vertex {j} is {g[j].tolist()!r}, "
                                 f"want {w[j].tolist()!r}")


def _check_raw(verts, coff, icoff, seg_off, what):
    """V = S + C, C <= S/4, every contour closed and at least 4 segments long, both offset arrays
    monotone from 0 to their totals, and each instance's contours holding its segments."""
    S, C, V = int(seg_off[-1]), int(icoff[-1]), len(verts)
    assert V == S + C and C <= S // 4, f"{what}: V={V} S={S} C={C}"
    assert len(coff) == C + 1 and coff[0] == 0 and coff[-1] == V, f"{what}: contour offsets"
    assert icoff[0] == 0 and (np.diff(icoff) >= 0).all(), f"{what}: instance contour offsets"
    assert (np.diff(coff) >= 5).all(), f"{what}: a contour of fewer than 4 segments"
    assert np.array_equal(verts[coff[:-1]], verts[coff[1:] - 1]), f"{what}: a contour not closed"
    held = np.concatenate([[0], np.cumsum(np.diff(coff) - 1)])[icoff]
    assert np.array_equal(held, seg_off), f"{what}: contour segments per instance"


def _device():
    import torch

    return torch.device("cuda", torch.cuda.current_device())


def _trace_engine(b):
    """engine.trace_packed_contours over batch b: (per image, per traced instance, the polygons;
    the number of contours in the buffers)."""
    import torch

    dev = _device()
    planes, R = b["planes"], b["regions"].shape[1]
    layout = BatchLayout([[p.shape[1], p.shape[2]] * 2 + [0, 0, p.shape[1], p.shape[2]]
                          for p in planes], R, limits=False)
    packed = np.zeros(int(layout.packed_off[-1]), np.uint8)
    for i, p in enumerate(planes):
        lo, hi = layout.packed_span(i, R)
        packed[lo:hi] = np.packbits(p, axis=-1).ravel()       # pad bits zero
    bufs = {}
    d_vert, d_coff, icoff = trace_packed_contours(
        N.load(), dev, torch.from_numpy(packed).to(dev),
        torch.from_numpy(np.ascontiguousarray(layout.packed_off)).to(dev),
        torch.tensor(b["counts"], dtype=torch.int32, device=dev),
        torch.from_numpy(layout.geom).to(dev),
        torch.from_numpy(np.ascontiguousarray(b["regions"])).to(dev), layout, bufs=bufs)
    verts, coff = _download_contours(d_vert, d_coff)
    _check_raw(verts, coff, icoff, bufs["inst"][:len(planes) * R + 1].cpu().numpy(),
               f"{b['name']} (engine)")
    return contours_to_lists(verts, coff, icoff, b["counts"], layout), int(icoff[-1])


def _trace_numpy(masks, boxes=None):
    """The NumPy entry's trace (visualize.mask_contours) of masks [H, W, n]; every box kept
    unless `boxes` says otherwise."""
    n = masks.shape[-1]
    bufs = {}
    layout, _, _, _, (d_vert, d_coff, _), icoff = visualize._trace_masks(
        np.ones((n, 4), np.int32) if boxes is None else boxes, masks, bufs)
    verts, coff = _download_contours(d_vert, d_coff)
    _check_raw(verts, coff, icoff, bufs["inst"][:n + 1].cpu().numpy(), "NumPy entry")
    return contours_to_lists(verts, coff, icoff, [n], layout)[0]


def _check_batch(b):
    """Batch b through the engine's trace, and each image's cut masks through the NumPy entry's
    with one more instance, a copy of the first under an all-zero box (no contour)."""
    got, n_contours = _trace_engine(b)
    total = 0
    for i, planes in enumerate(b["planes"]):
        n = b["counts"][i]
        cut = [E.cut(planes[k], b["regions"][i, k]) for k in range(n)]
        want = [E.reference(m, (0, 0) + m.shape) for m in cut]
        total += sum(len(w) for w in want)
        for k in range(n):
            _assert_same(got[i][k], want[k], f"{b['name']}: image {i}, instance {k} (engine)")
        if n:
            boxes = np.ones((n + 1, 4), np.int32)
            boxes[n] = 0
            mine = _trace_numpy(np.stack(cut + cut[:1], axis=-1), boxes)
            assert mine[n] == [], f"{b['name']}: image {i}: contours under an all-zero box"
            for k in range(n):
                _assert_same(mine[k], want[k], f"{b['name']}: image {i}, instance {k} (NumPy)")
    # instances past counts[b] hold set pixels: they are not traced
    assert n_contours == total, f"{b['name']}: {n_contours} contours traced, want {total}"


@pytest.mark.parametrize("name", ["seams", "placed saddles"])
def test_saddles_on_word_and_chunk_seams(cuda_device, name):
    """A: checkerboards, noise and lone saddles at window positions 0, 1, 32, 33 and on the
    1024-cell chunk seam, for every x1 mod 8."""
    for b in E.BUILDERS[name]()["batches"]:
        _check_batch(b)


def test_cut_regions(cuda_device):
    """B: regions outside the image on each side, empty, 1 x 1 and whole over planes set
    everywhere; 24 images of different sizes, B*R = 288; and a batch with nothing to trace."""
    for b in E.cut_regions()["batches"]:
        _check_batch(b)


def test_cycle_lengths_around_the_jump_rounds(cuda_device):
    """C: one call per L in {2^k - 2, 2^k, 2^k + 2}, k = 3..17, L the longest instance; and an
    instance of 16 384 segments whose cycles are all 4 long."""
    for b in E.jump_rounds()["batches"]:
        _check_batch(b)


def test_totals_and_heads_on_scan_tiles(cuda_device):
    """D: S in {4094, 4096, 4098, 8192, 4096 t +- 2}, cycle heads on segments 4094 and 4096."""
    for b in E.scan_tiles()["batches"]:
        _check_batch(b)


def test_checkerboard_of_2_25_segments(cuda_device):
    """D: a 4096 x 4096 checkerboard: 2^25 segments, 2^23 contours, 8192 scan tiles and 25
    jump rounds, its raw buffers against the closed form (no split into 8 M arrays)."""
    import torch

    S = 1 << 25
    need = N.contour_scratch_bytes(S) + 16 * (S + S // 4) + (1 << 24) * 2
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / GB:.1f} GB of free device memory; {free / GB:.1f} GB are free")
    m = E.checkerboard(4096, 4096, 1)
    bufs = {}
    _, _, _, _, (d_vert, d_coff, _), icoff = visualize._trace_masks(
        np.ones((1, 4), np.int32), m[:, :, None], bufs)
    del m
    seg_off = bufs["inst"][:2].cpu().numpy()
    assert seg_off.tolist() == [0, S] and icoff.tolist() == [0, S // 4]
    verts, coff = _download_contours(d_vert, d_coff)
    del d_vert, d_coff, bufs
    want_v, want_off = E.checkerboard_polygons(4096, 4096, 1)
    assert np.array_equal(coff, want_off)
    bad = np.flatnonzero((verts != want_v).any(axis=1))
    assert bad.size == 0, f"vertex {bad[0]} is {verts[bad[0]].tolist()}, want {want_v[bad[0]].tolist()}"


@pytest.mark.parametrize("case", E.long_masks(), ids=lambda c: c[0])
def test_vertices_exact_past_2_23(cuda_device, case):
    """E: thin masks of 2^23 + 40 and 2^24 + 40 pixels with pixels at both ends: halves past 2^23
    and odd integers past 2^24, which float32 rounds.  Through the engine's trace on packed
    planes, and through the NumPy entry where it packs the mask (mrx_pack_masks takes at most
    65535 rows)."""
    name, mask, blobs = case
    want = E.far_apart_reference(mask, blobs)
    b = E.batch(name, [mask[None]], [[(0, 0) + mask.shape]])
    _assert_same(_trace_engine(b)[0][0][0], want, f"{name} (engine)")
    if mask.shape[0] <= 65535:
        _assert_same(_trace_numpy(mask[:, :, None])[0], want, f"{name} (NumPy trace)")
        _assert_same(visualize.mask_contours(np.ones((1, 4), np.int32), mask[:, :, None])[0],
                     want, f"{name} (mask_contours)")


def test_engine_region_past_2_23(cuda_device):
    """E: a 2 x (2^23 + 40) plane of noise, traced in a box at its right end."""
    W = (1 << 23) + 40
    rng = np.random.default_rng(1105)
    plane = E.noise(rng, 2, W)
    region = (0, W - 37, 2, W)
    b = E.batch("2 x (2^23 + 40), box at the right end", [plane[None]], [[region]])
    got = _trace_engine(b)[0][0][0]
    want = E.reference(plane, region)
    assert want and want[-1][:, 0].max() > 1 << 23
    _assert_same(got, want, b["name"])
