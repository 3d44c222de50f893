"""mrx_poly_decode at the edges where its bit-exact claim can break (inputs:
tests/polygon_edge_inputs.py): every builder's annotations through MaskBatch.from_coco, the
planes equal to np.packbits of the oracle's masks bit for bit and the areas and extents the
oracle's; the same through evaluate.ann_to_mask and mixed into a batch next to RLE; and one image
of H*W >= 2^31 compared on the device with the oracle's runs given to from_rle."""
import numpy as np
import pytest
import torch

import polygon_edge_inputs as pe
import polygon_oracle as po
from bbox_oracle import extract_bboxes
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import evaluate
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import BatchLayout, MaskBatch

pytestmark = pytest.mark.gpu


def _geom(H, W):
    return [H, W, H, W, 0, 0, H, W]


def _dev():
    return torch.device("cuda", torch.cuda.current_device())


def _from_coco(images):
    geoms = [_geom(H, W) for (H, W), _ in images]
    segms = [s for _, s in images]
    gt = MaskBatch.from_coco(N.load(), _dev(), geoms, [np.ones(len(s), np.int32) for s in segms],
                             segms)
    layout = BatchLayout(gt.geom, gt.R, limits=False)
    packed = gt.planes.d_packed.cpu().numpy()
    planes = [packed[slice(*layout.packed_span(b, gt.counts[b]))].reshape(
        layout.packed_shape(b, gt.counts[b])) for b in range(gt.n)]
    return planes, gt.planes.d_areas.cpu().numpy(), gt.planes.d_extents.cpu().numpy()


def _mask(segm, H, W):
    if isinstance(segm, dict):
        return po.decode(segm["counts"], H, W)
    return po.ann_to_mask(segm, H, W, window=True)


def _check(images, want_from=None):
    """from_coco of `images` against the oracle's masks of `want_from` (default: the same)."""
    planes, areas, ext = _from_coco(images)
    for b, ((H, W), segms) in enumerate(want_from or images):
        for k, segm in enumerate(segms):
            m = _mask(segm, H, W)
            want = np.packbits(m, axis=-1)
            bad = np.argwhere(np.unpackbits(planes[b][k], axis=-1)[:, :W] != m)
            assert not bad.size, (f"image {b} ({H}x{W}), instance {k}: {len(bad)} pixels differ, "
                                  f"first (y, x) = {tuple(bad[0])}", segm)
            assert np.array_equal(planes[b][k], want), (b, k)   # pad bits too
            assert areas[b, k] == m.sum(), (b, k)
            assert np.array_equal(ext[b, k], extract_bboxes(m[:, :, None])[0]), (b, k)


@pytest.fixture(scope="module")
def built():
    return {b.__name__: b() for b in pe.BUILDERS}


@pytest.mark.parametrize("name", [b.__name__ for b in pe.BUILDERS])
def test_planes_equal_oracle(cuda_device, built, name):
    _check(built[name]["images"])


@pytest.mark.parametrize("name", ["unfused_minor", "toggle_rows", "scaling_ties", "box_lists",
                                  "int_range", "overlapping_parts"])
def test_ann_to_mask(cuda_device, built, name):
    for (H, W), segms in built[name]["images"][:6]:
        for segm in segms:
            got = evaluate.ann_to_mask({"segmentation": segm}, H, W)
            assert np.array_equal(got, _mask(segm, H, W).astype(np.uint8)), segm


@pytest.mark.parametrize("name", ["toggle_rows", "scan_seams", "y_major", "dense_toggles"])
def test_mixed_with_rle(cuda_device, built, name):
    """Every other instance given as the oracle's uncompressed runs: the polygon planes next to
    RLE planes in one batch are still the oracle's."""
    images = built[name]["images"]
    mixed = [((H, W), [segm if k % 2 else {"size": [H, W],
                                          "counts": po.ann_to_rle(segm, H, W, window=True)}
                       for k, segm in enumerate(segms)]) for (H, W), segms in images]
    _check(mixed, images)


def test_big_image_equals_rle_on_the_device(cuda_device):
    """H*W >= 2^31: pycocotools' int positions would overflow; the oracle's exact Python-int runs
    through from_rle give the planes from_coco gives, compared on the device."""
    ((H, W), segms), = pe.big_image()["images"]
    rles = [{"size": [H, W], "counts": po.ann_to_rle(s, H, W, window=True)} for s in segms]
    assert max(sum(r["counts"][:-1]) for r in rles) > 1 << 31
    cls = [np.ones(len(segms), np.int32)]
    a = MaskBatch.from_coco(N.load(), _dev(), [_geom(H, W)], cls, [segms])
    b = MaskBatch.from_rle(N.load(), _dev(), [_geom(H, W)], cls, [rles])
    # every byte of the planes; the slot's alignment padding after them is never written
    end = BatchLayout([_geom(H, W)], a.R, limits=False).packed_span(0, a.R)[1]
    assert a.R == b.R and end >= a.planes.d_packed.numel() - 15
    assert torch.equal(a.planes.d_packed[:end], b.planes.d_packed[:end])
    assert torch.equal(a.planes.d_areas, b.planes.d_areas)
    assert torch.equal(a.planes.d_extents, b.planes.d_extents)
