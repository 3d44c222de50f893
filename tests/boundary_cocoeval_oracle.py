"""CPU restatement of boundary_iou_api's COCOeval for iouType "boundary" (Cheng et al., "Boundary
IoU", CVPR 2021): `mask_to_boundary` calling the real cv2 as that API does, `_prepare` adding each
instance's boundary, and `computeIoU` taking np.minimum of rleIou on the masks and rleIou on the
boundaries, both with the iscrowd flags.  `evaluateImg`, `accumulate` and `summarize` are segm's,
so this is `cocoeval_oracle.COCOevalOracle` with `_prepare` and `computeIoU` replaced (a
detection's area stays its mask's pixel count).  TEST INFRASTRUCTURE ONLY.

*** PARITY UNPINNED ***  boundary_iou_api is not vendored or installed; this restates its
published code.  Inputs are those of `cocoeval_oracle`, and its stated difference applies.
"""
import numpy as np

from cocoeval_oracle import COCOevalOracle, Params, rle_iou  # noqa: F401  (Params: re-exported)


def dilation_of(h, w, dilation_ratio=0.02):
    """mask_to_boundary's dilation for an h x w image."""
    img_diag = np.sqrt(h ** 2 + w ** 2)
    dilation = int(round(dilation_ratio * img_diag))
    if dilation < 1:
        dilation = 1
    return dilation


def mask_to_boundary(mask, dilation_ratio=0.02):
    """boundary_iou_api's mask_to_boundary: uint8 [h, w] mask minus its erosion, cv2's."""
    import cv2

    mask = np.asarray(mask).astype(np.uint8)
    h, w = mask.shape
    dilation = dilation_of(h, w, dilation_ratio)
    new_mask = cv2.copyMakeBorder(mask, 1, 1, 1, 1, cv2.BORDER_CONSTANT, value=0)
    kernel = np.ones((3, 3), dtype=np.uint8)
    new_mask_erode = cv2.erode(new_mask, kernel, iterations=dilation)
    mask_erode = new_mask_erode[1: h + 1, 1: w + 1]
    return mask - mask_erode


def closed_form_boundary(mask, d):
    """mask AND NOT (the pixels whose (2d+1) x (2d+1) square lies inside the image and is all
    set), by a summed-area table of the mask padded with d zeros."""
    m = np.asarray(mask, bool)
    h, w = m.shape
    p = np.zeros((h + 2 * d + 1, w + 2 * d + 1), np.int64)
    p[1 + d:1 + d + h, 1 + d:1 + d + w] = m
    s = p.cumsum(0).cumsum(1)
    k = 2 * d + 1
    # the square of padded rows y .. y + 2d and columns x .. x + 2d: pixel (y, x)'s
    win = s[k:, k:] - s[:-k, k:] - s[k:, :-k] + s[:-k, :-k]
    return m & ~(win == k * k)


class COCOevalBoundaryOracle(COCOevalOracle):
    def __init__(self, gts, dts, params=None, dilation_ratio=0.02):
        super().__init__(gts, dts, params)
        self.dilation_ratio = dilation_ratio

    def _prepare(self):
        super()._prepare()
        for objs in list(self._gts.values()) + list(self._dts.values()):
            for o in objs:
                o["boundary"] = mask_to_boundary(o["mask"], self.dilation_ratio).astype(bool)

    def computeIoU(self, imgId, catId):
        p = self.params
        gt = self._gts[imgId, catId]
        dt = self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in inds]
        if len(dt) > p.maxDets[-1]:
            dt = dt[0:p.maxDets[-1]]
        if len(gt) == 0 or len(dt) == 0:
            return []
        mask_ious = np.zeros((len(dt), len(gt)))
        boundary_ious = np.zeros((len(dt), len(gt)))
        for di, d in enumerate(dt):
            for gi, g in enumerate(gt):
                mask_ious[di, gi] = rle_iou(d["mask"], g["mask"], int(g["iscrowd"]))
                boundary_ious[di, gi] = rle_iou(d["boundary"], g["boundary"], int(g["iscrowd"]))
        return np.minimum(mask_ious, boundary_ious)
