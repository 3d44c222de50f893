"""CPU restatement of pycocotools' COCOeval for iouType "bbox": `maskApi.c` `bbIou` loop for loop,
`computeIoU` on the `bbox` fields, and `loadRes`' `area = bb[2]*bb[3]` for detections.
`evaluateImg`, `accumulate` and `summarize` are the same for every IoU type, so this is
`cocoeval_oracle.COCOevalOracle` with `_prepare` and `computeIoU` replaced.  TEST INFRASTRUCTURE
ONLY.

*** PARITY UNPINNED ***  pycocotools is not vendored or installed; this restates its published
code.  Inputs are plain lists instead of COCO objects:

    gts: dicts {"image_id", "category_id", "bbox" ([x, y, w, h]), "iscrowd", "area"}
    dts: dicts {"image_id", "category_id", "bbox", "score"}, in results order

Python floats are IEEE doubles and every operation rounds on its own, as pycocotools' x86-64 C
build does.  The stated difference of `cocoeval_oracle` (matches recorded as positions) applies.
"""
from collections import defaultdict

import numpy as np

from cocoeval_oracle import COCOevalOracle, Params  # noqa: F401  (Params: re-exported)


def bb_iou(dt, gt, iscrowd):
    """maskApi.c bbIou: o[d][g] for boxes dt [m][4] and gt [n][4] ([x, y, w, h], float64)."""
    m, n = len(dt), len(gt)
    o = np.zeros((m, n))
    for g in range(n):
        G = [float(v) for v in gt[g]]
        ga = G[2] * G[3]
        crowd = iscrowd is not None and bool(iscrowd[g])
        for d in range(m):
            D = [float(v) for v in dt[d]]
            da = D[2] * D[3]
            o[d, g] = 0
            w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
            if w <= 0:
                continue
            h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
            if h <= 0:
                continue
            i = w * h
            u = da if crowd else da + ga - i
            o[d, g] = i / u
    return o


class COCOevalBboxOracle(COCOevalOracle):
    def _prepare(self):
        p = self.params
        self._gts = defaultdict(list)
        self._dts = defaultdict(list)
        for gid, g in enumerate(self.gts_in):
            if g["image_id"] in p.imgIds and g["category_id"] in p.catIds:
                g = dict(g, id=gid)
                g["ignore"] = g.get("iscrowd", 0)
                self._gts[g["image_id"], g["category_id"]].append(g)
        for did, d in enumerate(self.dts_in):
            if d["image_id"] in p.imgIds and d["category_id"] in p.catIds:
                bb = d["bbox"]
                d = dict(d, id=did, iscrowd=0, area=bb[2] * bb[3])
                self._dts[d["image_id"], d["category_id"]].append(d)

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
        g = [x["bbox"] for x in gt]
        d = [x["bbox"] for x in dt]
        iscrowd = [int(o["iscrowd"]) for o in gt]
        return bb_iou(d, g, iscrowd)
