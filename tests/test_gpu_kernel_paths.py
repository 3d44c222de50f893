"""The two byte-canvas expand kernels against each other, and the launches around them.

`mrx_mask_expand` takes the team kernel while a tile row of R instances fits a team's buffer and
the generic kernel beyond that (or for mask tiles wider than 30 columns).  Both compute the one
sample of expand.cuh, so the same instances must give the same canvas byte for byte, whichever
kernel runs and however the generic kernel cuts the canvas into chunks.  Padding an image's
detection rows with class-0 rows (`pad_rows`) changes R and nothing else, so it picks the
kernel without changing the answer."""
import random

import numpy as np
import pytest

import contour_oracle as co
import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import sharding, synth, visualize

from helpers import (canvas_masks, check_values, compare_masks, oracle_unmold, pad_rows,
                     prepared_engine, record_stats)

pytestmark = pytest.mark.gpu

GENERIC_R = 320      # no team buffer holds a tile row of 320 instances


def _expand(ims, R, classes, mask_hw=28, poison=True, **kw):
    """Engine after prepare + expand of `ims` padded to R rows; returns (engine, counts)."""
    eng = prepared_engine([pad_rows(im, R) for im in ims], R, classes, np.float32, mask_hw, **kw)
    if poison:
        eng.d_canvas.fill_(7)            # every byte of the result must be rewritten
    eng.enqueue_expand()
    counts = eng.fetch_meta()[0].copy()
    return eng, counts


def _assert_same_canvas(a, b, counts, what):
    import torch

    for i in range(len(counts)):
        H, W = (int(v) for v in a._geom_host[i][:2])
        assert tuple(b._geom_host[i][:2]) == (H, W)
        n = H * W * int(counts[i])
        oa, ob = int(a._offsets[i]), int(b._offsets[i])
        assert torch.equal(a.d_canvas[oa:oa + n], b.d_canvas[ob:ob + n]), f"{what}: image {i}"


# ------------------------------------------------------------------------ team == generic
@pytest.mark.parametrize("name,hw,n,R,mask_hw,zero_area", [
    ("28x28", (240, 333), 90, 100, 28, ()),
    ("14x16", (240, 333), 90, 100, (14, 16), ()),
    ("33x24", (240, 333), 90, 100, (33, 24), ()),
    ("coco_unaligned_zero_area", (800, 1333), 90, 100, 28, (2, 50, 89)),
    ("two_cull_passes", (800, 1333), 150, 160, 28, (0, 129)),
])
def test_team_and_generic_kernels_write_the_same_bytes(cuda_device, name, hw, n, R, mask_hw,
                                                       zero_area):
    rng = np.random.default_rng(808)
    ims = [synth.make_image(rng, hw, n, num_classes=4, max_instances=R, mask_hw=mask_hw,
                            min_box=1, max_box_frac=1.0 if k else 0.5,
                            zero_area_rows=zero_area)
           for k in range(2)]
    team, counts = _expand(ims, R, 4, mask_hw)
    generic, counts_g = _expand(ims, GENERIC_R, 4, mask_hw)
    assert np.array_equal(counts, counts_g)
    if zero_area:
        assert (counts < n).all()        # rows were dropped: instance k is not tile k
    _assert_same_canvas(team, generic, counts, name)


def _values_supported(im, R):
    """True when mrx_mask_expand_values takes R rows (the team kernel fits).  An unsupported R
    is refused before anything is launched."""
    import torch

    eng = prepared_engine([pad_rows(im, R)], R, 3, np.float32)
    d_values = torch.empty(int(eng._offsets[1]), dtype=torch.float32, device="cuda")
    try:
        eng.enqueue_expand_values(d_values)
    except N.MrxError as e:
        assert "status -2" in str(e), e
        return False
    return True


def test_team_kernel_largest_R(cuda_device):
    """Find R*, the largest R the team kernel takes for one image, by bisection through the
    values entry point.  At R* the samples are within tolerance; R* + 1 takes the generic kernel
    and writes the same bytes."""
    rng = np.random.default_rng(809)
    im = synth.make_image(rng, (240, 333), 90, num_classes=3, max_instances=90, min_box=1,
                          max_box_frac=1.0)
    lo, hi = 100, GENERIC_R
    assert _values_supported(im, lo) and not _values_supported(im, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _values_supported(im, mid):
            lo = mid
        else:
            hi = mid
    r_star = lo
    record_stats("team_kernel_largest_R", {"B": 1, "R_star": r_star})
    print(f"team kernel largest R at B = 1: {r_star}")
    # entries pack the instance and its tile index into 8 bits each
    assert r_star <= 256
    check_values(f"values/R{r_star}", [pad_rows(im, r_star)], r_star, 3, np.float32)
    at, counts = _expand([im], r_star, 3)
    above, counts_above = _expand([im], r_star + 1, 3)
    assert np.array_equal(counts, counts_above)
    _assert_same_canvas(at, above, counts, f"R = {r_star} vs {r_star + 1}")


# ------------------------------------------------------------------------ generic-kernel chunks
def _largest_chunk(mw, B):
    """Largest chunk_bytes whose shared-memory footprint fits a CTA of the generic kernel: the
    chunk, two staged tile rows and one 48-byte entry for each of 64 entries, the job prefix, and
    256 bytes for the kernel's static shared memory."""
    import torch

    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    return (optin - 64 * 2 * mw * 4 - 64 * 48 - (B + 1) * 4 - 256) // 16 * 16


def test_generic_kernel_chunks_and_ctas(cuda_device):
    """The generic kernel cuts each canvas into flat chunks of chunk_bytes; at N = 250 most chunk
    sizes split a pixel's N bytes between two chunks.  Every cut and CTA count gives the bytes of
    the default launch."""
    rng = np.random.default_rng(810)
    ims = [synth.make_image(rng, (300, 421), 250, num_classes=4, max_instances=GENERIC_R,
                            min_box=1, max_box_frac=1.0 if k else 0.3) for k in range(2)]
    ref, counts = _expand(ims, GENERIC_R, 4)
    assert (counts > 200).all()
    chunks = [1024, 1040, 4112, 25600, 51200, _largest_chunk(28, len(ims))]
    for chunk in chunks:
        for ctas in (0, 1):
            eng, c = _expand(ims, GENERIC_R, 4, chunk_bytes=chunk, ctas_per_sm=ctas)
            assert np.array_equal(c, counts)
            _assert_same_canvas(ref, eng, counts, f"chunk_bytes={chunk} ctas_per_sm={ctas}")


# ------------------------------------------------------------------------ mixed geometries
MIXED = [((17, 9), 5), ((333, 517), 30), ((800, 1333), 0), ((1024, 1024), 45), ((64, 2048), 20)]


@pytest.fixture(scope="module")
def mixed_batch():
    """One batch of five original shapes, each with its own molded window, ragged counts
    (one image has none), and the oracle's answer for each image."""
    rng = np.random.default_rng(811)
    ims = [synth.make_image(rng, hw, n, num_classes=4, max_instances=100, min_box=1,
                            max_box_frac=1.0) for hw, n in MIXED]
    refs = [oracle_unmold(im, np.float32, return_resized=True) for im in ims]
    return ims, refs


@pytest.mark.parametrize("R", [100, GENERIC_R], ids=["team", "generic"])
def test_expand_launches_after_one_prepare(cuda_device, mixed_batch, R):
    """Every expand launch leaves its scheduler words at zero for the next one (mrx.h,
    MRX_SCHED_WORDS): after one prepare, expanding the batch in image ranges, one launch each,
    writes the bytes of a single launch.  One range holds only the image without instances."""
    ims, _ = mixed_batch
    whole, counts = _expand(ims, R, 4)
    eng = prepared_engine([pad_rows(im, R) for im in ims], R, 4, np.float32)
    eng.d_canvas.fill_(7)
    bounds = sharding.chunk_bounds(len(ims), 3)
    assert len(bounds) == 3 and (2, 3) in bounds and counts[2] == 0
    for b0, b1 in bounds:
        eng.enqueue_expand(images=(b0, b1))
    _assert_same_canvas(whole, eng, counts, f"launches over {bounds}")


@pytest.mark.parametrize("R", [100, GENERIC_R], ids=["team", "generic"])
def test_mixed_geometries_in_one_launch(cuda_device, mixed_batch, R):
    ims, refs = mixed_batch
    eng, counts = _expand(ims, R, 4)
    _, boxes, cls, scores = eng.fetch_meta()
    masks = []
    for b, (im, (rb, rc, rs, rm, rz)) in enumerate(zip(ims, refs)):
        k = int(counts[b])
        assert k == rb.shape[0]
        np.testing.assert_array_equal(boxes[b, :k], rb)
        np.testing.assert_array_equal(cls[b, :k], rc)
        np.testing.assert_array_equal(scores[b, :k], rs)
        m = canvas_masks(eng, b, k)
        if k:
            assert compare_masks(m, rm, rz, rb)[0] == 0, f"image {b}"
        masks.append(m)
    assert counts[2] == 0 and (np.delete(counts, 2) > 0).all()

    def check_packed(d_packed, off, what):
        for b, im in enumerate(ims):
            H, W = im.original_image_shape[:2]
            k, wb = int(counts[b]), (W + 7) // 8
            got = d_packed[int(off[b]):int(off[b]) + k * H * wb].cpu().numpy().reshape(k, H, wb)
            assert np.array_equal(got, np.packbits(masks[b].transpose(2, 0, 1), axis=-1)), \
                f"{what}: image {b}"

    d_packed, off = eng.enqueue_expand_packed()
    check_packed(d_packed, off, "mrx_mask_expand_packed")
    d_packed.fill_(0xAA)
    check_packed(*eng.pack_masks(), "mrx_pack_masks")

    # contours of those planes; B * R > 1024 for the generic R, so the instance offsets are
    # scanned in more than one pass of the one-CTA scan
    polys = eng.enqueue_contours()
    for b in range(len(ims)):
        k = int(counts[b])
        want = co.mask_polygons(boxes[b, :k], masks[b])
        assert len(polys[b]) == k == len(want), f"contours: image {b}"
        for n, (got, ref) in enumerate(zip(polys[b], want)):
            assert len(got) == len(ref) and all(np.array_equal(g, r) for g, r in zip(got, ref)), \
                f"contours: image {b}, instance {n}"

    d_runs, off = eng.enqueue_rle()
    runs = d_runs.cpu().numpy().view(np.uint32)
    for b in range(len(ims)):
        for n in range(int(counts[b])):
            i = b * R + n
            want = oracle.rle_encode(masks[b][:, :, n])["counts"]
            assert np.array_equal(runs[int(off[i]) + i:int(off[i + 1]) + i + 1], want), (b, n)

    img_rng = np.random.default_rng(812)
    images = [synth.synth_rgb_image(img_rng, *im.original_image_shape[:2]) for im in ims]
    colors = [visualize.random_colors(R, rng=random.Random(20 + b)) for b in range(len(ims))]
    outs = visualize.composite_batch(eng, images, colors)
    for b in range(len(ims)):
        k = int(counts[b])
        want = oracle.composite_instances(images[b], boxes[b, :k], masks[b], colors[b]) \
            if k else images[b]
        assert np.array_equal(outs[b].cpu().numpy(), want), f"composite: image {b}"
