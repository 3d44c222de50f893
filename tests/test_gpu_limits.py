"""The unmold kernels at the size limits they accept, against the float64 oracle.

The other suites check every kernel on small inputs.  Here each limit that `engine.plan` and
include/mrx.h promise is reached:

  1. tile tickets: launches of the team kernel on both sides of the point where its tile counter
     changes from float to integer tickets, and the scheduler words it leaves between them;
  2. 64-bit offsets: canvas slots and packed planes that straddle or lie past 2^31 and 2^32 bytes;
  3. the largest single image: 2^30 pixels (team kernel, packed planes, RLE, strings, contours)
     and H*W*R just below 2^31 - 2^20 bytes (generic kernel);
  4. the largest batch: MRX_MAX_BATCH images through every entry point, and the team kernel's
     largest R at that batch size;

and one past each limit is refused before anything is launched.

At these sizes the oracle's `unmold_detections`, which builds [H, W, N] arrays on the host, is too
expensive, so groups 1-3 check each instance inside its box only ("box-local"): the device bytes
of canvas[y1:y2, x1:x2, n] against `oracle.resize(tile, (y2 - y1, x2 - x1)) >= 0.5` with the band
rule of `helpers.compare_masks`, and a device count of the instance's whole plane equal to the
in-box count, so that nothing is set outside the box.  Boxes are exact pixel boxes on unscaled
molds with float64 detections; the oracle's box arithmetic must reproduce them bit for bit.

Every group reads `torch.cuda.mem_get_info()` while its buffers are allocated and records the
device memory it used with `record_stats` (canvases come from mrx_device_alloc, which torch's
allocator statistics do not see)."""
import gc
import random

import numpy as np
import pytest

import contour_oracle as co
import oracle
from coco_oracle import rle_to_string
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import synth, visualize
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import UnmoldEngine, make_geom

from helpers import (check_values, compare_masks, oracle_unmold, pad_rows, prepared_engine,
                     record_stats, tile_hw)

pytestmark = pytest.mark.gpu

POISON = 0x5A            # canvas / packed bytes no kernel writes (masks are 0 / 1)
GB = 1e9


# ------------------------------------------------------------------------ shared helpers
@pytest.fixture(autouse=True)
def _release_device_memory():
    """Each test frees its engines (and the canvases mrx_device_alloc gave them) before the next."""
    yield
    import torch

    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


class _Memory:
    """Device memory a group uses: free memory at its start minus the lowest seen since."""

    def __init__(self, name):
        import torch

        torch.cuda.synchronize()
        self.name = name
        self.free0 = torch.cuda.mem_get_info()[0]
        self.used = 0

    def sample(self):
        import torch

        torch.cuda.synchronize()
        self.used = max(self.used, self.free0 - torch.cuda.mem_get_info()[0])

    def record(self, **extra):
        record_stats(f"limits_memory/{self.name}", {"device_bytes": int(self.used), **extra})
        print(f"{self.name}: {self.used / GB:.2f} GB of device memory")


def _require_free(nbytes, what):
    import torch

    free = torch.cuda.mem_get_info()[0]
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / GB:.1f} GB of free device memory; "
                    f"{free / GB:.1f} GB are free")


def _exact_image(rng, hw, boxes, R, mask_hw=28, classes=3):
    """An image on an unscaled mold (molded pixels are original pixels) whose detections are the
    pixel `boxes` in float64, random class ids in [1, classes) and random mask tiles; rows past
    the boxes are class-0 padding."""
    H, W = hw
    mh, mw = tile_hw(mask_hw)
    det = np.zeros((R, 6), np.float64)
    n = len(boxes)
    if n:
        px = np.asarray(boxes, np.float64)
        det[:n, :4] = (px - [0, 0, 1, 1]) / [H - 1, W - 1, H - 1, W - 1]
        det[:n, 4] = rng.integers(1, classes, n)
        det[:n, 5] = 0.9
    msk = rng.random((R, mh, mw, classes), dtype=np.float32)
    im = synth.SynthImage(det, msk, (H, W, 3), (H, W, 3), (0, 0, H, W), n)
    kept, rows = _oracle_boxes(im)
    assert [tuple(int(v) for v in b) for b in kept] == [tuple(b) for b in boxes], \
        "the oracle's box arithmetic must give the pixel boxes back"
    assert list(rows) == list(range(n))
    return im


def _holds_poison(t):
    """True when every byte of device tensor `t` is still POISON.  (A plain bool: pytest would
    otherwise explain a failed `==` on a tensor element by element.)"""
    return bool(t.eq(POISON).all())


def _count_set(t):
    """Nonzero bytes of a 2-D device view, counted in blocks of rows (a whole 2^30-byte plane at
    once would take gigabytes of temporaries)."""
    import torch

    return sum(int(torch.count_nonzero(t[r:r + 4096])) for r in range(0, t.shape[0], 4096))


def _oracle_boxes(im):
    """Steps 1-6 of the oracle's unmold_detections (trim, window normalisation, box affine,
    denorm, zero-area drop) without the masks: (kept boxes int32 [N, 4], their detection rows)."""
    det = im.detections
    zero = np.where(det[:, 4] == 0)[0]
    n = zero[0] if zero.shape[0] else det.shape[0]
    wy1, wx1, wy2, wx2 = oracle.norm_boxes(np.asarray(im.window), im.image_shape[:2])
    shift = np.array([wy1, wx1, wy1, wx1])
    scale = np.array([wy2 - wy1, wx2 - wx1, wy2 - wy1, wx2 - wx1])
    boxes = oracle.denorm_boxes(np.divide(det[:n, :4] - shift, scale), im.original_image_shape[:2])
    keep = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1]) > 0
    return boxes[keep], np.flatnonzero(keep)


def _tile(im, row):
    """float64 class tile of detection row `row` (what the device expands, widened)."""
    return im.mrcnn_mask[row, :, :, int(im.detections[row, 4])].astype(np.float64)


def _engine(ims, R, mask_hw=28, canvas=True):
    """UnmoldEngine planned for `ims` (float64 detections, float32 masks) after prepare + class
    gather; no mask has been expanded.  The device boxes must be the oracle's."""
    import torch

    eng = UnmoldEngine(len(ims), R, tile_hw(mask_hw), ims[0].mrcnn_mask.shape[-1],
                       det_dtype=np.float64, mask_dtype=np.float32)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims],
             canvas=canvas)
    d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
    eng.enqueue(d_det, d_msk, expand=False)
    return eng


def _check_meta(eng, ims):
    counts, boxes = eng.fetch_meta()[:2]
    for b, im in enumerate(ims):
        want = _oracle_boxes(im)[0]
        assert int(counts[b]) == len(want), f"image {b}"
        assert np.array_equal(boxes[b, :len(want)], want), f"image {b}"
    return counts.copy()


def _check_local(got, tile, box):
    """One instance inside its box: host bytes `got` [y2 - y1, x2 - x1] (0 / 1) against the
    oracle's resize of its tile, with the band rule of compare_masks.  Returns the set pixels."""
    y1, x1, y2, x2 = (int(v) for v in box)
    z = oracle.resize(tile, (y2 - y1, x2 - x1))
    got = np.asarray(got)
    assert got.shape == z.shape, (got.shape, z.shape)
    assert int(got.max(initial=0)) <= 1, f"box {box}: bytes other than 0 / 1"
    g = got.astype(np.bool_)[:, :, None]
    bad, _ = compare_masks(g, (z >= 0.5)[:, :, None], [z], [(0, 0, y2 - y1, x2 - x1)])
    assert bad == 0, f"box {box}: {bad} pixels differ from the oracle outside the band"
    return int(g.sum())


def _check_canvas(eng, b, im, ks=None):
    """Box-local check of image b's byte canvas, instances `ks` (default: all).  Returns
    {k: bool [y2 - y1, x2 - x1]} of the device masks inside their boxes."""
    import torch

    boxes, rows = _oracle_boxes(im)
    view = eng.canvas_view(b, len(boxes))
    local = {}
    for k in (range(len(boxes)) if ks is None else ks):
        y1, x1, y2, x2 = (int(v) for v in boxes[k])
        got = view[y1:y2, x1:x2, k].cpu().numpy()
        n = _check_local(got, _tile(im, rows[k]), boxes[k])
        assert _count_set(view[:, :, k]) == n, \
            f"image {b}, instance {k}: bytes set outside its box"
        local[k] = got.astype(np.bool_)
    return local


def _packed_plane(eng, b, k):
    """uint8 device view [H, ceil(W/8)] of instance k's packed plane in image b."""
    H, W = (int(v) for v in eng._geom_host[b][:2])
    wb = (W + 7) // 8
    o = int(eng.packed_layout()[0][b]) + k * H * wb
    return eng.d_packed[o:o + H * wb].view(H, wb)


def _check_packed(eng, b, im, ks):
    """Box-local check of instances `ks` of image b's packed planes: the bits inside the box
    against the oracle, every bit outside it zero.  Returns {k: bool in-box mask}."""
    import torch

    boxes, rows = _oracle_boxes(im)
    local = {}
    for k in ks:
        y1, x1, y2, x2 = (int(v) for v in boxes[k])
        plane = _packed_plane(eng, b, k)
        c0, c1 = x1 // 8, (x2 + 7) // 8
        rect = plane[y1:y2, c0:c1]
        bits = np.unpackbits(rect.cpu().numpy(), axis=1)
        lo, hi = x1 - 8 * c0, x2 - 8 * c0
        assert not bits[:, :lo].any() and not bits[:, hi:].any(), f"image {b}, instance {k}"
        _check_local(bits[:, lo:hi], _tile(im, rows[k]), boxes[k])
        assert _count_set(plane) == _count_set(rect), \
            f"image {b}, instance {k}: bits set outside its box"
        local[k] = bits[:, lo:hi].astype(np.bool_)
    return local


def _local_polygons(local, box):
    """The contour polygons display_instances draws for a mask that is zero outside `box`,
    from its in-box part: the contour oracle on the box, shifted to image coordinates."""
    y1, x1 = int(box[0]), int(box[1])
    polys = co.mask_polygons(np.ones((1, 4), np.int32), local[:, :, None])[0]
    return [v + np.array([x1, y1], np.float64) for v in polys]


def _same_polygons(got, want, what):
    assert len(got) == len(want), f"{what}: {len(got)} contours, want {len(want)}"
    for i, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), f"{what}: contour {i}"


# ------------------------------------------------------------------------ 1. tile tickets
# expand_team.cu: launch_expand_team ships teams of 6 x 5 warps building tiles of 10 canvas rows,
# one CTA per SM.  mask_expand_team_kernel draws FLOAT tickets while the launch has fewer than
# 2^24 - 4 * SMs * 6 tiles (`float_tickets`) and integer tickets from there on.  tile_geom gives a
# tile P = W pixels wide when a tile row holds the whole image row, so an image 2 pixels wide has
# ceil(H / 10) tiles when it has instances and none when it has not.
TEAMS = 6
TILE_ROWS = 10
TALL_W, TALL_R = 2, 2
# (H, boxes): distinct heights and box positions; the last variant has no instances (no tiles)
TALL_VARIANTS = [
    (65530, [(0, 0, 1400, 2), (30000, 1, 31234, 2)]),
    (65521, [(64000, 0, 65521, 1)]),
    (64007, [(100, 0, 2100, 2), (63000, 0, 64007, 2)]),
    (65535, [(1, 0, 65535, 2)]),
    (4001, []),
]


def _tiles(H, n):
    return -(-H // TILE_ROWS) if n else 0


def _float_ticket_limit():
    import torch

    return (1 << 24) - 4 * torch.cuda.get_device_properties(0).multi_processor_count * TEAMS


def _alone_bytes(im, R, mask_hw=28):
    """The canvas bytes [H, W, N] of `im` planned alone at offset 0, checked box-locally against
    the oracle: the expected bytes of every copy of the image in a batch."""
    eng = _engine([im], R, mask_hw)
    eng.d_canvas.fill_(POISON)
    eng.enqueue_expand()
    n = _check_meta(eng, [im])[0]
    _check_canvas(eng, 0, im)
    H, W = im.original_image_shape[:2]
    return eng.d_canvas[:H * W * int(n)].clone()


@pytest.fixture(scope="module")
def tall_variants():
    """The variants as images, with their expected canvas bytes on the device."""
    rng = np.random.default_rng(4001)
    ims = [_exact_image(rng, (H, TALL_W), boxes, TALL_R) for H, boxes in TALL_VARIANTS]
    return ims, [_alone_bytes(im, TALL_R) for im in ims]


def _tall_batch(rng, variants, target):
    """Images cycling through the variants, then one more whose height makes the launch's tile
    count exactly `target`.  Returns (images, expected bytes per image)."""
    ims, want = variants
    seq, total = [], 0
    while True:
        v = len(seq) % len(ims)
        t = _tiles(ims[v].original_image_shape[0], ims[v].n_valid)
        if total + t >= target:
            break
        seq.append(v)
        total += t
    r = target - total                  # 1 <= r <= 6554 tiles left: H = 10 r - 5 <= 65535 rows
    H = TILE_ROWS * r - 5
    last = _exact_image(rng, (H, TALL_W), [(max(1, H // 3), 0, H - 1, TALL_W)], TALL_R)
    batch = [ims[v] for v in seq] + [last]
    assert len(batch) <= N.MRX_MAX_BATCH
    assert sum(_tiles(im.original_image_shape[0], im.n_valid) for im in batch) == target
    return batch, [want[v] for v in seq] + [_alone_bytes(last, TALL_R)]


def _check_tall(eng, batch, want, b0=0, b1=None):
    """Every byte of every [H_b, W_b, N_b] prefix of images [b0, b1) equals the expected bytes;
    the slots of images without instances still hold the poison."""
    import torch

    canvas, off = eng.d_canvas, eng._offsets
    for b in range(b0, len(batch) if b1 is None else b1):
        o = int(off[b])
        n = want[b].numel()
        if n:
            assert torch.equal(canvas[o:o + n], want[b]), f"image {b}"
        else:
            assert _holds_poison(canvas[o:int(off[b + 1])]), f"image {b} was written"


TICKET_TARGETS = ["T*-1", "T*", "2^24-1", "2^24", "2^24+1", "2^24+1e5"]


def _target(name):
    t_star = _float_ticket_limit()
    return {"T*-1": t_star - 1, "T*": t_star, "2^24-1": (1 << 24) - 1, "2^24": 1 << 24,
            "2^24+1": (1 << 24) + 1, "2^24+1e5": (1 << 24) + 100000}[name]


@pytest.mark.parametrize("target", TICKET_TARGETS)
def test_tile_tickets_around_the_float_counter_limit(cuda_device, tall_variants, target):
    """A launch of exactly T tiles writes every tile once, whichever ticket format T selects:
    T* - 1 is the last launch with float tickets, T* the first with integer ones."""
    _require_free(2 * GB, "a batch of 2^24 tiles")
    mem = _Memory(f"tickets/{target}")
    T = _target(target)
    batch, want = _tall_batch(np.random.default_rng(4002), tall_variants, T)
    eng = _engine(batch, TALL_R)
    counts = _check_meta(eng, batch)
    assert sum(_tiles(im.original_image_shape[0], int(c)) for im, c in zip(batch, counts)) == T
    eng.d_canvas.fill_(POISON)
    eng.enqueue_expand()
    mem.sample()
    _check_tall(eng, batch, want)
    mem.record(images=len(batch), tiles=T)


def test_scheduler_words_between_float_and_integer_launches(cuda_device, tall_variants):
    """Every launch leaves the scheduler words zeroed in either ticket format: after one prepare
    (which zeroes them itself), launches over image ranges below and above the float limit
    alternate, and each writes the bytes of a fresh launch."""
    _require_free(2 * GB, "a batch of 2^24 tiles")
    t_star = _float_ticket_limit()
    batch, want = _tall_batch(np.random.default_rng(4003), tall_variants, (1 << 24) + 100000)
    eng = _engine(batch, TALL_R)
    counts = _check_meta(eng, batch)
    tiles = np.array([_tiles(im.original_image_shape[0], int(c)) for im, c in zip(batch, counts)])
    h = len(batch) // 2
    assert tiles[:h].sum() < t_star and tiles[h:].sum() < t_star and tiles.sum() >= t_star
    # float, integer, float, integer
    for rng_ in [(h, len(batch)), (0, len(batch)), (0, h), (0, len(batch))]:
        eng.d_canvas.fill_(POISON)
        eng.enqueue_expand(images=rng_)
        _check_tall(eng, batch, want, *rng_)


# ------------------------------------------------------------------------ 2. past 2^31 / 2^32
# BASELINE.json configs[3]: 2160x3840 images at R = 50, 414.72 MB of canvas per slot
BIG_HW = (2160, 3840)


def _random_boxes(rng, hw, n, lo, hi):
    H, W = hw
    out = []
    for _ in range(n):
        bh, bw = (int(v) for v in rng.integers(lo, hi + 1, 2))
        y1, x1 = int(rng.integers(0, H - bh + 1)), int(rng.integers(0, W - bw + 1))
        out.append((y1, x1, y1 + bh, x1 + bw))
    return out


def _boundary_box(hw, N, slot_off, boundary):
    """A box across the canvas rows where byte `boundary` of the buffer falls inside an image at
    `slot_off` with N instances."""
    H, W = hw
    row = (boundary - slot_off) // N // W
    assert 0 <= row < H
    return (max(0, row - 40), 100, min(H, row + 40), W - 100)


@pytest.mark.parametrize("kernel,mask_hw", [("team", (28, 28)), ("generic", (28, 32))])
def test_canvas_slots_past_2_31_and_2_32_bytes(cuda_device, kernel, mask_hw):
    """12 slots of configs[3]: image 5 straddles 2^31, image 10 straddles 2^32 and image 11 lies
    past it; they have detections, the other slots are reserved and never written.  The probes'
    canvas, packed planes and overlay equal those of the same image planned alone at offset 0."""
    import torch

    R, B = 50, 12
    slot = BIG_HW[0] * BIG_HW[1] * R
    _require_free(8 * GB, "12 canvases of 2160x3840x50")
    mem = _Memory(f"offsets/{kernel}")
    rng = np.random.default_rng(4010)
    probes = {5: 1 << 31, 10: 1 << 32, 11: 1 << 32}
    assert 5 * slot < (1 << 31) < 6 * slot and 10 * slot < (1 << 32) < 11 * slot
    ims = []
    for b in range(B):
        boxes = []
        if b in probes:
            boxes = [_boundary_box(BIG_HW, R, b * slot, probes[b])] if b != 11 else []
            boxes += _random_boxes(rng, BIG_HW, R - len(boxes), 8, 1200)
        ims.append(_exact_image(rng, BIG_HW, boxes, R, mask_hw))
    eng = _engine(ims, R, mask_hw)
    assert [int(v) for v in eng._offsets] == [b * slot for b in range(B + 1)]
    counts = _check_meta(eng, ims)
    assert all(int(counts[b]) == (R if b in probes else 0) for b in range(B))
    eng.d_canvas.fill_(POISON)
    eng.enqueue_expand()
    eng._packed_buffer()
    eng.d_packed.fill_(POISON)
    eng.pack_masks()
    img = np.random.default_rng(4011).integers(0, 256, BIG_HW + (3,), dtype=np.uint8)
    colors = visualize.random_colors(R, rng=random.Random(4012))
    outs = visualize.composite_batch(eng, [img] * B, colors)
    mem.sample()

    d_img = torch.from_numpy(img).cuda()
    poff = eng.packed_layout()[0]
    for b in range(B):
        if b not in probes:
            assert _holds_poison(eng.d_canvas[b * slot:(b + 1) * slot]), \
                f"filler slot {b} was written"
            assert _holds_poison(eng.d_packed[int(poff[b]):int(poff[b + 1])]), \
                f"filler packed slot {b} was written"
            assert torch.equal(outs[b], d_img), f"overlay of filler {b}"
            continue
        _check_canvas(eng, b, ims[b], ks=[0, 1, R // 2, R - 1])
        alone = _engine([ims[b]], R, mask_hw)
        alone.d_canvas.fill_(POISON)
        alone.enqueue_expand()
        alone.pack_masks()
        alone_out = visualize.composite_batch(alone, [img], colors)[0]
        assert torch.equal(eng.d_canvas[b * slot:(b + 1) * slot], alone.d_canvas[:slot]), \
            f"canvas of image {b}"
        n = int(poff[b + 1] - poff[b])
        assert torch.equal(eng.d_packed[int(poff[b]):int(poff[b]) + n], alone.d_packed[:n]), \
            f"packed planes of image {b}"
        assert torch.equal(outs[b], alone_out), f"overlay of image {b}"
        mem.sample()
        alone.release()
        del alone, alone_out
    mem.record(canvas_bytes=B * slot)


def test_packed_planes_past_2_32_bytes(cuda_device):
    """With no byte canvas (plan(canvas=False)), 21 packed slots of 2160x3840 at R = 200
    (207.36 MB each): image 10 straddles 2^31 and image 20 straddles 2^32.
    mrx_mask_expand_packed and the contours of the probes equal those of the same image planned
    alone.  (mrx_pack_masks writing past 2^32 would need about 34 GB of byte canvas to read
    from; it is left out.)"""
    import torch

    R, B = 200, 21
    _require_free(6 * GB, "21 packed slots of 2160x3840x200")
    mem = _Memory("offsets/packed")
    rng = np.random.default_rng(4020)
    wb = (BIG_HW[1] + 7) // 8
    pslot = R * BIG_HW[0] * wb
    probes = {10: 1 << 31, 20: 1 << 32}
    ims = [_exact_image(rng, BIG_HW, _random_boxes(rng, BIG_HW, R, 4, 300) if b in probes else [],
                        R) for b in range(B)]
    eng = _engine(ims, R, canvas=False)
    assert eng.d_canvas is None
    poff, total = eng.packed_layout()
    assert [int(v) for v in poff] == [b * pslot for b in range(B + 1)]
    counts = _check_meta(eng, ims)
    eng._packed_buffer()
    eng.d_packed.fill_(POISON)
    eng.enqueue_expand_packed()
    polys = eng.enqueue_contours()
    mem.sample()
    for b in range(B):
        if b not in probes:
            assert int(counts[b]) == 0 and polys[b] == []
            assert _holds_poison(eng.d_packed[int(poff[b]):int(poff[b + 1])]), \
                f"filler packed slot {b} was written"
            continue
        assert int(counts[b]) == R
        k_cross = (probes[b] - int(poff[b])) // (BIG_HW[0] * wb)      # plane across the boundary
        ks = sorted({0, k_cross - 1, k_cross, k_cross + 1, R - 1})
        local = _check_packed(eng, b, ims[b], ks)
        boxes = _oracle_boxes(ims[b])[0]
        for k in ks:
            _same_polygons(polys[b][k], _local_polygons(local[k], boxes[k]),
                           f"image {b}, instance {k}")
        alone = _engine([ims[b]], R, canvas=False)
        d_alone, _ = alone.enqueue_expand_packed()
        alone_polys = alone.enqueue_contours()[0]
        assert torch.equal(eng.d_packed[int(poff[b]):int(poff[b + 1])], d_alone[:pslot]), \
            f"packed planes of image {b}"
        for k in range(R):
            _same_polygons(polys[b][k], alone_polys[k], f"image {b}, instance {k} vs alone")
        mem.sample()
        alone.release()
        del alone, d_alone
    mem.record(packed_bytes=int(total))


# ------------------------------------------------------------------------ 3. the largest image
def _runs_from_box(local, box, H, W):
    """COCO run lengths of an [H, W] mask that is zero outside `box` (y1 > 0), from its in-box
    part: the column-major positions of its value changes, never a 2^30-element array."""
    y1, x1, y2, x2 = (int(v) for v in box)
    assert y1 > 0           # every column enters the box from a zero pixel
    d = np.diff(np.pad(local.astype(np.int8), ((1, 1), (0, 0))), axis=0)   # [h + 1, w]
    j, i = np.nonzero(d.T)                                                # column-major order
    pos = (x1 + j.astype(np.int64)) * H + y1 + i
    pos = pos[pos < H * W]  # a run open at the last pixel of the image ends with it
    return np.diff(np.concatenate([[0], pos, [H * W]])).astype(np.uint32)


def _count_lengths(s):
    """Characters of each count of a compressed RLE string (0x20 marks a continued count)."""
    out, cur = [], 0
    for c in s:
        cur += 1
        if not (c - 48) & 0x20:
            out.append(cur)
            cur = 0
    assert cur == 0
    return out


def test_team_kernel_at_2_30_pixels(cuda_device):
    """One 32768x32768 image (R = 1, 1 GiB of canvas) with its box in the last rows and columns,
    where flat offsets are largest: byte canvas, packed expand, pack_masks, RLE, strings and
    contours.  The leading zero run is longer than 2^29 pixels, so its count takes 7 characters."""
    import torch

    H = W = 1 << 15
    _require_free(3 * GB, "a 2^30-pixel canvas")
    mem = _Memory("largest_image/team")
    box = (H - 1200, W - 1500, H, W)
    im = _exact_image(np.random.default_rng(4030), (H, W), [box], 1)
    eng = _engine([im], 1)
    assert int(eng._offsets[1]) == 1 << 30
    _check_meta(eng, [im])
    eng.d_canvas.fill_(POISON)
    eng.enqueue_expand()
    local = _check_canvas(eng, 0, im)[0]
    assert local.any() and not local.all()

    d_packed, _ = eng.enqueue_expand_packed()
    mem.sample()
    assert np.array_equal(_check_packed(eng, 0, im, [0])[0], local)
    expanded = d_packed[:H * (W // 8)].clone()
    d_packed.fill_(POISON)
    eng.pack_masks()
    mem.sample()
    assert torch.equal(eng.d_packed[:H * (W // 8)], expanded), "pack_masks != packed expand"
    del expanded

    want = _runs_from_box(local, box, H, W)
    assert want[0] >= 1 << 29 and int(want.astype(np.int64).sum()) == H * W
    d_runs, off = eng.enqueue_rle()
    assert np.array_equal(d_runs[int(off[0]):int(off[1]) + 1].cpu().numpy().view(np.uint32), want)
    d_str, d_str_off = eng.enqueue_rle_strings()
    so = d_str_off.cpu().numpy()
    s = bytes(d_str[int(so[0]):int(so[1])].cpu().numpy())
    assert s == rle_to_string(want)
    assert _count_lengths(s)[0] == 7
    mem.sample()

    polys = eng.enqueue_contours()
    _same_polygons(polys[0][0], _local_polygons(local, box), "contours")
    mem.record()


def test_generic_kernel_at_the_byte_limit(cuda_device):
    """H*W*R within 2^20 of the largest canvas plan() accepts (2^31 - 2^20 bytes), through the
    generic kernel (tiles 32 columns wide), with boxes in the last rows where its 32-bit chunk
    offsets are largest."""
    H, W, R = 1 << 15, (1 << 15) - 17, 2
    limit = (1 << 31) - (1 << 20)
    assert limit - (1 << 20) <= H * W * R < limit
    _require_free(3 * GB, "a canvas of 2^31 - 2^20 bytes")
    mem = _Memory("largest_image/generic")
    boxes = [(H - 1500, W - 1900, H, W), (H - 800, 40, H - 5, 1800)]
    im = _exact_image(np.random.default_rng(4031), (H, W), boxes, R, mask_hw=(28, 32))
    eng = _engine([im], R, mask_hw=(28, 32))
    _check_meta(eng, [im])
    eng.d_canvas.fill_(POISON)
    eng.enqueue_expand()
    mem.sample()
    _check_canvas(eng, 0, im)
    mem.record()


# ------------------------------------------------------------------------ 4. the largest batch
MAX_B = N.MRX_MAX_BATCH
BATCH_R = 16             # MRX_MAX_BATCH * 16 = 65 536 instance slots through the one-CTA scans
BATCH_HS = (2, 3, 5, 8, 13, 21, 29, 40)
BATCH_WS = (2, 3, 7, 12, 19, 33, 50, 70)


def _max_batch_images(seed, mask_hw, R=BATCH_R):
    """MRX_MAX_BATCH small images cycling through shapes 2x2 .. 40x70; every third image (b % 3
    == 1) has no detections, the last one has some."""
    rng = np.random.default_rng(seed)
    ims = []
    for b in range(MAX_B):
        hw = (BATCH_HS[b % len(BATCH_HS)], BATCH_WS[(b // len(BATCH_HS)) % len(BATCH_WS)])
        n = 0 if b % 3 == 1 else int(rng.integers(1, R + 1))
        ims.append(synth.make_image(rng, hw, n, num_classes=3, max_instances=R, mask_hw=mask_hw,
                                    min_box=1, max_box_frac=1.0))
    return ims


def _oracle_batch(ims):
    return [oracle_unmold(im, np.float32, return_resized=True) for im in ims]


def _host_masks(eng, counts, refs):
    """Per image, the bool [H, W, N] host masks of the byte canvas, checked against the oracle."""
    host = eng.d_canvas[:int(eng._offsets[-1])].cpu().numpy()
    masks = []
    for b, (rb, rc, rs, rm, rz) in enumerate(refs):
        H, W = (int(v) for v in eng._geom_host[b][:2])
        k = int(counts[b])
        o = int(eng._offsets[b])
        m = host[o:o + H * W * k].reshape(H, W, k)
        assert int(m.max(initial=0)) <= 1, f"image {b}: bytes other than 0 / 1"
        m = m.astype(np.bool_)
        assert k == rb.shape[0], f"image {b}"
        if k:
            assert compare_masks(m, rm, rz, rb)[0] == 0, f"image {b}"
        masks.append(m)
    return masks


@pytest.fixture(scope="module")
def max_batch():
    ims = _max_batch_images(4040, (12, 12))
    return ims, _oracle_batch(ims)


def test_max_batch_every_entry_point(cuda_device, max_batch):
    """MRX_MAX_BATCH images through prepare, the team expand, the packed expand, pack_masks, RLE,
    strings, contours and the overlay, each image against the full oracle."""
    import torch

    ims, refs = max_batch
    mem = _Memory("max_batch")
    eng = prepared_engine(ims, BATCH_R, 3, np.float32, (12, 12))
    counts, boxes, cls, scores = eng.fetch_meta()
    counts = counts.copy()
    assert counts[MAX_B - 1] > 0 and (counts[1::3] == 0).all()
    for b, (rb, rc, rs, rm, rz) in enumerate(refs):
        k = int(counts[b])
        assert k == rb.shape[0], f"image {b}"
        np.testing.assert_array_equal(boxes[b, :k], rb)
        np.testing.assert_array_equal(cls[b, :k], rc)
        np.testing.assert_array_equal(scores[b, :k], rs)
    eng.d_canvas.fill_(POISON)
    eng.enqueue_expand()
    masks = _host_masks(eng, counts, refs)

    def check_packed(d_packed, off, what):
        host = d_packed.cpu().numpy()
        for b, m in enumerate(masks):
            H, W, k = m.shape
            wb = (W + 7) // 8
            got = host[int(off[b]):int(off[b]) + k * H * wb].reshape(k, H, wb)
            assert np.array_equal(got, np.packbits(m.transpose(2, 0, 1), axis=-1)), \
                f"{what}: image {b}"

    d_packed, off = eng.enqueue_expand_packed()
    check_packed(d_packed, off, "mrx_mask_expand_packed")
    d_packed.fill_(POISON)
    check_packed(*eng.pack_masks(), "mrx_pack_masks")

    d_runs, ioff = eng.enqueue_rle()
    runs = d_runs.cpu().numpy().view(np.uint32)
    d_str, d_str_off = eng.enqueue_rle_strings()
    strs, soff = d_str.cpu().numpy(), d_str_off.cpu().numpy()
    assert len(ioff) == len(soff) == MAX_B * BATCH_R + 1
    for b, m in enumerate(masks):
        for n in range(m.shape[2]):
            i = b * BATCH_R + n
            want = oracle.rle_encode(m[:, :, n])["counts"]
            assert np.array_equal(runs[int(ioff[i]) + i:int(ioff[i + 1]) + i + 1], want), (b, n)
            assert bytes(strs[int(soff[i]):int(soff[i + 1])]) == rle_to_string(want), (b, n)
        for n in range(m.shape[2], BATCH_R):
            assert soff[b * BATCH_R + n] == soff[b * BATCH_R + n + 1]

    polys = eng.enqueue_contours()
    for b, m in enumerate(masks):
        k = m.shape[2]
        want = co.mask_polygons(boxes[b, :k], m)
        assert len(polys[b]) == k == len(want), f"contours: image {b}"
        for n, (got, ref) in enumerate(zip(polys[b], want)):
            _same_polygons(got, ref, f"contours: image {b}, instance {n}")

    img_rng = np.random.default_rng(4041)
    images = [img_rng.integers(0, 256, im.original_image_shape, dtype=np.uint8) for im in ims]
    colors = visualize.random_colors(BATCH_R, rng=random.Random(4042))
    outs = visualize.composite_batch(eng, images, colors)
    mem.sample()
    host_outs = [o.cpu().numpy() for o in outs]
    for b, m in enumerate(masks):
        k = m.shape[2]
        want = oracle.composite_instances(images[b], boxes[b, :k], m, colors) if k else images[b]
        assert np.array_equal(host_outs[b], want), f"composite: image {b}"
    del outs
    torch.cuda.synchronize()
    mem.record()


def test_max_batch_generic_kernel(cuda_device):
    """MRX_MAX_BATCH images through the generic kernel (tiles 32 columns wide)."""
    ims = _max_batch_images(4050, (8, 32))
    refs = _oracle_batch(ims)
    eng = prepared_engine(ims, BATCH_R, 3, np.float32, (8, 32))
    counts = eng.fetch_meta()[0].copy()
    eng.d_canvas.fill_(POISON)
    eng.enqueue_expand()
    _host_masks(eng, counts, refs)


def _team_takes(ims, R):
    """True when the team kernel takes R rows for this batch (mrx_mask_expand_values refuses an R
    it cannot take with MRX_E_UNSUPPORTED before launching anything)."""
    import torch

    eng = prepared_engine([pad_rows(im, R) for im in ims], R, 3, np.float32, (2, 4))
    d_values = torch.empty(int(eng._offsets[len(ims)]), dtype=torch.float32, device="cuda")
    try:
        eng.enqueue_expand_values(d_values)
    except N.MrxError as e:
        assert "status -2" in str(e), e
        return False
    return True


def _largest_team_R(ims):
    lo, hi = 100, 320
    assert _team_takes(ims, lo) and not _team_takes(ims, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _team_takes(ims, mid):
            lo = mid
        else:
            hi = mid
    return lo


def test_team_kernel_largest_R_at_max_batch(cuda_device):
    """R*, the team kernel's largest R, at B = MRX_MAX_BATCH (its scheduler table takes shared
    memory from the tile buffers): no larger than at B = 1, within 1e-6 of the oracle at R*, and
    R* + 1 takes the generic kernel and writes the same bytes."""
    import torch

    ims = _max_batch_images(4060, (2, 4), R=8)
    r_one = _largest_team_R(ims[:1])
    r_max = _largest_team_R(ims)
    record_stats("team_kernel_largest_R", {"B": 1, "R_star": r_one})
    record_stats("team_kernel_largest_R", {"B": MAX_B, "R_star": r_max})
    print(f"team kernel largest R: {r_one} at B = 1, {r_max} at B = {MAX_B}")
    assert r_max <= r_one
    check_values(f"values/B{MAX_B}/R{r_max}", [pad_rows(im, r_max) for im in ims], r_max, 3,
                 np.float32, (2, 4))
    engs = []
    for R in (r_max, r_max + 1):
        eng = prepared_engine([pad_rows(im, R) for im in ims], R, 3, np.float32, (2, 4))
        eng.d_canvas.fill_(POISON)
        eng.enqueue_expand()
        engs.append((eng, eng.fetch_meta()[0].copy()))
    (at, counts), (above, counts_above) = engs
    assert np.array_equal(counts, counts_above)
    for b in range(MAX_B):
        H, W = (int(v) for v in at._geom_host[b][:2])
        n = H * W * int(counts[b])
        oa, ob = int(at._offsets[b]), int(above._offsets[b])
        assert torch.equal(at.d_canvas[oa:oa + n], above.d_canvas[ob:ob + n]), f"image {b}"


# ------------------------------------------------------------------------ one past each limit
def _geom(H, W):
    return make_geom((H, W, 3), (H, W, 3), (0, 0, H, W))


@pytest.mark.parametrize("limit", ["batch", "pixels", "bytes"])
def test_one_past_each_limit_is_refused(cuda_device, limit):
    """The engine refuses one image too many, an image of 2^30 + 1 pixels and a canvas of
    H*W*R = 2^31 - 2^20 bytes before it allocates or launches anything, and takes the largest
    accepted size.  (mrx_mask_expand's own MRX_E_INVALID for B > MRX_MAX_BATCH is checked in
    test_host.py, without a device.)"""
    if limit == "batch":
        with pytest.raises(ValueError):
            UnmoldEngine(MAX_B + 1, 8, (2, 4), 2)
        eng = UnmoldEngine(MAX_B, 1, (2, 4), 2)
        with pytest.raises(ValueError):
            eng.plan([_geom(2, 2)] * (MAX_B + 1))
        assert eng.d_canvas is None and eng._n_images == 0
        eng.plan([_geom(2, 2)] * MAX_B)
        assert eng._n_images == MAX_B
        return
    if limit == "pixels":
        R, refused, accepted = 1, (5, 214748365), (1 << 15, 1 << 15)
        assert refused[0] * refused[1] == (1 << 30) + 1
    else:
        # 2^31 - 2^20 = 32768 * 32752 * 2 bytes is refused; 2^31 - 2^20 - 1 = 13919 * 51403 * 3
        R, refused, accepted = 2, (1 << 15, 32752), (13919, 51403)
        assert refused[0] * refused[1] * R == (1 << 31) - (1 << 20)
        assert accepted[0] * accepted[1] * 3 == (1 << 31) - (1 << 20) - 1
    eng = UnmoldEngine(1, R, (2, 4), 2)
    with pytest.raises(ValueError):
        eng.plan([_geom(*refused)])
    assert eng.d_canvas is None and eng._n_images == 0
    eng = UnmoldEngine(1, R if limit == "pixels" else 3, (2, 4), 2)
    eng.plan([_geom(*accepted)], canvas=False)
    assert eng._n_images == 1 and eng.d_canvas is None
