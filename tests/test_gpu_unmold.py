"""GPU parity of api_utils.unmold_detections (serve.py:147-154) against the oracle.

Contract (SURVEY.md 8c): N, boxes, class_ids, scores bit-exact; binary masks equal
wherever the oracle's float64 pre-threshold value is > 1e-6 away from 0.5.  That is the claim
against upstream's float64; the claim against the fp32 sample the kernels define
(csrc/expand.cuh), bit for bit with no band, is test_gpu_expand_exact.py's.
"""
import numpy as np
import pytest

import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, synth
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import UnmoldEngine, make_geom

from helpers import (MASK_VALUE_ATOL, check_values, compare_masks, item_of, oracle_unmold,
                     run_with_values)

pytestmark = pytest.mark.gpu


def _check_image(im, dtype):
    ref_b, ref_c, ref_s, ref_m, resized = oracle_unmold(im, dtype, return_resized=True)
    b, c, s, m = api_utils.unmold_detections(*item_of(im, dtype))
    assert b.dtype == np.int32 and c.dtype == np.int32
    np.testing.assert_array_equal(b, ref_b)
    np.testing.assert_array_equal(c, ref_c)
    assert s.dtype == ref_s.dtype
    np.testing.assert_array_equal(s, ref_s)
    bad, band = compare_masks(m, ref_m, resized, ref_b)
    assert bad == 0, f"{bad} mask pixels differ outside the +-{MASK_VALUE_ATOL} band"
    return band


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("hw,n,classes", [
    ((1024, 1024), 10, 81),      # BASELINE.json config 1 shape
    ((96, 128), 12, 5),
    ((800, 1333), 37, 81),       # COCO shape: rows not 16-byte aligned, ragged N
    ((333, 517), 100, 2),        # tiny-class case, odd sizes
])
def test_unmold_matches_oracle(cuda_device, hw, n, classes, dtype):
    im = synth.make_batch(11, 1, hw, n, num_classes=classes)[0]
    _check_image(im, dtype)


def test_trim_at_first_zero_class_and_zero_area(cuda_device):
    rng = np.random.default_rng(5)
    # original == molded size (scale 1) so x2 == x1 in molded pixels stays zero-width
    im = synth.make_image(rng, (1024, 1024), 20, num_classes=7, zero_area_rows=(0, 7, 19))
    im.detections[15, 4] = 0.0      # early class-0 row truncates; rows 16.. ignored
    ref = oracle_unmold(im)
    got = api_utils.unmold_detections(*item_of(im))
    assert got[0].shape[0] == ref[0].shape[0] == 13    # 15 rows minus zero-area rows 0 and 7
    for g, r in zip(got[:3], ref[:3]):
        np.testing.assert_array_equal(g, r)
    _check_image(im, np.float64)


def test_concurrent_callers_do_not_interleave(cuda_device):
    """api_utils is called from a threaded web server in the reference's deployment: two
    threads hammering the same cached engine with different images must each get their own
    image's result (the engine lock spans plan -> enqueue -> fetch)."""
    import threading

    ims = synth.make_batch(404, 2, (96, 128), 9, num_classes=4, max_instances=12)
    refs = [oracle_unmold(im, np.float32) for im in ims]
    errors = []

    def worker(i):
        try:
            for _ in range(25):
                b, c, s, m = api_utils.unmold_detections(*item_of(ims[i], np.float32))
                assert np.array_equal(b, refs[i][0]) and np.array_equal(m, refs[i][3])
        except BaseException as e:      # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


def test_no_detections(cuda_device):
    rng = np.random.default_rng(6)
    im = synth.make_image(rng, (64, 80), 0, num_classes=3)
    b, c, s, m = api_utils.unmold_detections(*item_of(im))
    rb, rc, rs, rm = oracle_unmold(im)
    assert b.shape == rb.shape == (0, 4) and c.shape == (0,) and s.shape == (0,)
    assert m.shape == rm.shape == (64, 80, 0) and m.dtype == rm.dtype


def test_leading_unit_batch_dim(cuda_device):
    im = synth.make_batch(3, 1, (120, 90), 6, num_classes=4)[0]
    it = item_of(im)
    got = api_utils.unmold_detections(it[0][None], it[1][None], *it[2:])
    ref = oracle_unmold(im)
    np.testing.assert_array_equal(got[0], ref[0])
    np.testing.assert_array_equal(got[3], ref[3])


@pytest.mark.parametrize("R,n", [(160, 160), (160, 131), (320, 300)])
def test_more_instances_than_one_cull_pass(cuda_device, R, n):
    """The team kernel culls 128 boxes per pass: N > 128 takes several passes over a tile;
    R = 320 does not fit its tile buffers at all and must fall back to the generic kernel."""
    rng = np.random.default_rng(77)
    im = synth.make_image(rng, (96, 128), n, num_classes=3, max_instances=R)
    _check_image(im, np.float64)


def test_every_box_meets_every_tile(cuda_device):
    """Adversarial density: 140 nearly canvas-sized boxes, every tile lists all of them."""
    rng = np.random.default_rng(78)
    im = synth.make_image(rng, (64, 96), 140, num_classes=3, max_instances=140,
                          min_box=60, max_box_frac=1.0)
    _check_image(im, np.float64)


@pytest.mark.parametrize("seed", range(24))
def test_random_shape_sweep(cuda_device, seed):
    """Seeded sweep over odd canvas sizes, instance counts and class counts: tile widths of
    1 .. 40 column blocks, aligned and unaligned rows, partial last tiles in both directions,
    boxes from 1 px to the whole window."""
    rng = np.random.default_rng(1000 + seed)
    H = int(rng.integers(17, 260))
    W = int(rng.integers(16, 420))
    R = int(rng.choice([1, 2, 3, 7, 16, 33, 64, 100]))
    n = int(rng.integers(0, R + 1))
    classes = int(rng.choice([2, 3, 81]))
    im = synth.make_image(rng, (H, W), n, num_classes=classes, max_instances=R,
                          min_box=1, max_box_frac=float(rng.choice([0.1, 0.5, 1.0])))
    dtype = np.float64 if seed % 2 else np.float32
    if n == 0:      # upstream returns np.empty((H, W, 0)) (float64), not a bool array
        got = api_utils.unmold_detections(*item_of(im, dtype))
        ref = oracle_unmold(im, dtype)
        assert got[3].shape == ref[3].shape == (H, W, 0) and got[3].dtype == ref[3].dtype
        assert got[0].shape == (0, 4)
        return
    _check_image(im, dtype)


def test_small_boxes_downscale(cuda_device):
    # boxes smaller than the 28x28 tile (no anti-aliasing in the reference)
    rng = np.random.default_rng(8)
    im = synth.make_image(rng, (150, 150), 30, num_classes=3, min_box=1, max_box_frac=0.1)
    _check_image(im, np.float64)


def test_batch_ragged_counts(cuda_device):
    ims = synth.make_batch(21, 5, (240, 320), (0, 40), num_classes=6, max_instances=40)
    got = api_utils.unmold_detections_batch([item_of(im) for im in ims])
    for im, g in zip(ims, got):
        rb, rc, rs, rm, rz = oracle_unmold(im, return_resized=True)
        np.testing.assert_array_equal(g[0], rb)
        np.testing.assert_array_equal(g[1], rc)
        np.testing.assert_array_equal(g[2], rs)
        if rb.shape[0]:
            assert compare_masks(g[3], rm, rz, rb)[0] == 0
        else:
            assert g[3].shape == rm.shape


@pytest.mark.parametrize("chunk", [1024, 4096, 20000 // 16 * 16, 51200])
def test_chunk_size_independent(cuda_device, chunk):
    """The canvas is cut into flat chunks; results must not depend on the cut."""
    import torch

    ims = synth.make_batch(31, 3, (130, 170), (5, 25), num_classes=4, max_instances=25)
    eng = UnmoldEngine(3, 25, (28, 28), 4, chunk_bytes=chunk)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims])
    d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
    eng.enqueue(d_det, d_msk)
    counts, boxes, cls, scores = eng.fetch_meta()
    for b, im in enumerate(ims):
        rb, rc, rs, rm, rz = oracle_unmold(im, np.float32, return_resized=True)
        k = int(counts[b])
        assert k == rb.shape[0]
        m = eng.canvas_view(b, k).cpu().numpy().view(np.bool_)
        assert compare_masks(m, rm, rz, rb)[0] == 0


@pytest.mark.parametrize("name,hw,n,R,classes,kw", [
    ("small_mixed", (96, 128), 12, 16, 5, {}),
    ("tiny_boxes_downscale", (150, 150), 30, 32, 3, dict(min_box=1, max_box_frac=0.1)),
    ("whole_canvas_boxes", (64, 96), 40, 40, 3, dict(min_box=60, max_box_frac=1.0)),
    ("coco_shape_unaligned", (800, 1333), 37, 100, 81, {}),
    ("odd_sizes_two_classes", (333, 517), 100, 100, 2, {}),
    ("more_than_one_cull_pass", (96, 128), 150, 160, 3, {}),
])
def test_production_kernel_values_within_tolerance(cuda_device, name, hw, n, R, classes, kw):
    """The stated fp32 tolerance, measured on the production kernel itself: every
    pre-threshold sample of every instance within 1e-6 of the float64 oracle."""
    rng = np.random.default_rng(909)
    ims = [synth.make_image(rng, hw, n, num_classes=classes, max_instances=R, **kw)
           for _ in range(2)]
    check_values("values/" + name, ims, R, classes)


def test_identity_resize_is_exact(cuda_device):
    """A 28x28 box is the identity resize: the samples equal the tile bit for bit."""
    rng = np.random.default_rng(4)
    im = synth.make_image(rng, (64, 64), 6, num_classes=3, max_instances=8, min_box=28,
                          max_box_frac=28 / 64, mold=((64, 64, 3), (0, 0, 64, 64)))
    (b, c, m, v), = run_with_values([im], 8, 3)
    assert ((b[:, 2] - b[:, 0]) == 28).all() and ((b[:, 3] - b[:, 1]) == 28).all()
    for i, (y1, x1, y2, x2) in enumerate(b):
        assert np.array_equal(v[y1:y2, x1:x2, i], im.mrcnn_mask[i, :, :, int(c[i])])


def test_exhaustive_config2_values_and_masks(cuda_device):
    """BASELINE.json configs[1] shape, EVERY instance of two images (1024x1024, 100 instances):
    values within 1e-6, masks equal outside the band; max error / band / flip counts recorded."""
    ims = synth.make_batch(77, 2, (1024, 1024), 100)
    tot = check_values("exhaustive/config2_2x1024x1024x100", ims, 100, 81)
    assert tot["instances"] == 200


def test_exhaustive_config4_4k(cuda_device):
    """BASELINE.json configs[3] shape, every instance of one 2160x3840 image (50 instances)."""
    ims = synth.make_batch(55, 1, (2160, 3840), 50, max_instances=50)
    tot = check_values("exhaustive/config4_1x2160x3840x50", ims, 50, 81)
    assert tot["instances"] == 50


def test_exhaustive_first_image_of_the_bench_batch(cuda_device):
    """The exact first image bench.py times (same seed, same generator call)."""
    import bench

    im = bench.make_bench_images(0, 1)[0]
    tot = check_values("exhaustive/bench_image0", [im], bench.N_INST, bench.CLASSES)
    assert tot["instances"] == bench.N_INST


def test_bad_class_id_raises_like_numpy(cuda_device):
    im = synth.make_batch(4, 1, (64, 64), 3, num_classes=3)[0]
    im.detections[1, 4] = 7.0
    with pytest.raises(IndexError):
        oracle_unmold(im)
    with pytest.raises(IndexError):
        api_utils.unmold_detections(*item_of(im))


def test_full_size_properties(cuda_device):
    """BASELINE.json config 2 shape (1024x1024, 100 instances) on a few images: values are
    0/1, support of instance n lies inside box n, and per-instance pixel counts equal the
    oracle's for a sampled subset of instances."""
    import torch

    ims = synth.make_batch(77, 4, (1024, 1024), 100)
    eng = UnmoldEngine(4, 100, (28, 28), 81)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims])
    d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
    eng.enqueue(d_det, d_msk)
    counts, boxes, cls, scores = eng.fetch_meta()
    for b, im in enumerate(ims):
        k = int(counts[b])
        assert k == 100
        v = eng.canvas_view(b, k)
        assert int(v.max()) <= 1
        per_inst = v.sum(dim=(0, 1), dtype=torch.int64).cpu().numpy()
        m = v.cpu().numpy().view(np.bool_)
        for i in range(0, k, 9):
            y1, x1, y2, x2 = boxes[b, i]
            assert m[:, :, i].sum() == m[y1:y2, x1:x2, i].sum() == per_inst[i]
            tile = im.mrcnn_mask[i, :, :, int(cls[b, i])].astype(np.float64)
            rz = oracle.resize(tile, (y2 - y1, x2 - x1))
            ref = rz >= 0.5
            d = m[y1:y2, x1:x2, i] != ref
            assert not (d & (np.abs(rz - 0.5) > MASK_VALUE_ATOL)).any()


@pytest.mark.parametrize("name", ["unmold_small", "unmold_coco_shape"])
def test_golden_fixture(cuda_device, name):
    """Committed fixture (tests/golden/make_golden.py): exact ints, masks equal outside the
    recorded +-1e-6 band around the threshold."""
    import os

    g = np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))
    b, c, s, m = api_utils.unmold_detections(
        g["detections"].astype(np.float64), g["mrcnn_mask"].astype(np.float64),
        tuple(g["original_image_shape"]), tuple(g["image_shape"]), tuple(g["window"]))
    np.testing.assert_array_equal(b, g["boxes"])
    np.testing.assert_array_equal(c, g["class_ids"])
    np.testing.assert_array_equal(s, g["scores"])
    shape = tuple(g["masks_shape"])
    want = np.unpackbits(g["masks_packed"])[:int(np.prod(shape))].reshape(shape).astype(bool)
    band = np.unpackbits(g["band_packed"])[:int(np.prod(shape))].reshape(shape).astype(bool)
    assert m.shape == shape
    assert not ((m != want) & ~band).any()


@pytest.mark.parametrize("hw,n,R,mask_hw", [((300, 421), 250, 320, 28), ((150, 203), 30, 40, 32)],
                         ids=["large_R", "wide_tiles"])
def test_generic_kernel_path(cuda_device, hw, n, R, mask_hw):
    """R = 320 detection rows do not fit the team kernel's tile buffers, and 32-column mask
    tiles do not fit a warp's lanes: the generic kernel takes over and must satisfy the same
    contract, on a canvas with unaligned rows and many tiles."""
    rng = np.random.default_rng(12)
    im = synth.make_image(rng, hw, n, num_classes=6, max_instances=R, mask_hw=mask_hw)
    _check_image(im, np.float64)


def test_config4_4k_shape_properties(cuda_device):
    """BASELINE.json config 4 shape: 3840x2160 original, 50 instances (one image here; the
    batch of 128 shards by image).  Support inside the box, per-instance parity with the
    oracle on a sample of instances, counts of ones computed on the device."""
    import torch

    ims = synth.make_batch(55, 2, (2160, 3840), 50, max_instances=50)
    eng = UnmoldEngine(2, 50, (28, 28), 81)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims])
    d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
    eng.enqueue(d_det, d_msk)
    counts, boxes, cls, scores = eng.fetch_meta()
    for b, im in enumerate(ims):
        k = int(counts[b])
        assert k == 50
        v = eng.canvas_view(b, k)
        assert int(v.max()) <= 1
        per_inst = v.sum(dim=(0, 1), dtype=torch.int64).cpu().numpy()
        # boxes: upstream's window / affine / denorm arithmetic on the same float32 rows
        wn = oracle.norm_boxes(np.array(im.window), im.image_shape[:2])
        shift = np.array([wn[0], wn[1], wn[0], wn[1]])
        scale = np.array([wn[2] - wn[0], wn[3] - wn[1], wn[2] - wn[0], wn[3] - wn[1]])
        ref_boxes = oracle.denorm_boxes(np.divide(im.detections[:k, :4] - shift, scale),
                                        im.original_image_shape[:2])
        np.testing.assert_array_equal(boxes[b, :k], ref_boxes)
        for i in range(0, k, 7):
            y1, x1, y2, x2 = boxes[b, i]
            sub = v[y1:y2, x1:x2, i].cpu().numpy().view(np.bool_)
            assert sub.sum() == per_inst[i]                      # nothing outside the box
            tile = im.mrcnn_mask[i, :, :, int(cls[b, i])].astype(np.float64)
            rz = oracle.resize(tile, (y2 - y1, x2 - x1))
            d = sub != (rz >= 0.5)
            assert not (d & (np.abs(rz - 0.5) > MASK_VALUE_ATOL)).any()


def test_config3_coco_batch_ragged(cuda_device):
    """BASELINE.json config 3 shape: 800x1333 originals, 1-100 instances per image (a batch
    of 6 here): row size not a multiple of 16 -> flat chunks; exact ints, masks vs oracle."""
    ims = synth.make_batch(66, 6, (800, 1333), (1, 100))
    got = api_utils.unmold_detections_batch([item_of(im, np.float32) for im in ims])
    for im, g in zip(ims, got):
        rb, rc, rs, rm, rz = oracle_unmold(im, np.float32, return_resized=True)
        np.testing.assert_array_equal(g[0], rb)
        np.testing.assert_array_equal(g[1], rc)
        np.testing.assert_array_equal(g[2], rs)
        assert compare_masks(g[3], rm, rz, rb)[0] == 0


def test_streaming_unmolder_pipeline(cuda_device):
    """engine.StreamingUnmolder: double-buffered H2D / D2H around the engine gives the same
    bytes as the plain call, batch after batch."""
    import torch

    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import StreamingUnmolder

    batches = [synth.make_batch(300 + k, 3, (160, 208), 20, num_classes=5, max_instances=20)
               for k in range(4)]
    geoms = [make_geom(im.original_image_shape, im.image_shape, im.window) for im in batches[0]]
    eng = UnmoldEngine(3, 20, (28, 28), 5)
    sm = StreamingUnmolder(eng, geoms)
    pinned = []
    for ims in batches:
        h_det = torch.from_numpy(np.stack([im.detections for im in ims])).pin_memory()
        h_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).pin_memory()
        pinned.append((h_det, h_msk))
    tickets = []
    results = {}
    for k, (h_det, h_msk) in enumerate(pinned):
        tickets.append(sm.submit(h_det, h_msk))
        if k:
            c, b, o = sm.wait(tickets[k - 1])
            results[k - 1] = (c.clone(), b.clone(), o.clone())
    c, b, o = sm.wait(tickets[-1])
    results[len(pinned) - 1] = (c.clone(), b.clone(), o.clone())
    for k, ims in enumerate(batches):
        counts, boxes, out = results[k]
        for i, im in enumerate(ims):
            rb, rc, rs, rm, rz = oracle_unmold(im, np.float32, return_resized=True)
            n = int(counts[i])
            assert n == rb.shape[0]
            np.testing.assert_array_equal(boxes[i, :n].numpy(), rb)
            off = int(eng._offsets[i])
            H, W = im.original_image_shape[:2]
            m = out[off:off + H * W * n].numpy().reshape(H, W, n).view(np.bool_)
            assert compare_masks(m, rm, rz, rb)[0] == 0
