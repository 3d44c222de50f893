"""CPU restatement of pycocotools' COCOeval for iouType "segm" (`cocoeval.py`: `_prepare`,
`computeIoU`, `evaluateImg`, `accumulate`, `summarize`; `maskApi.c`: `rleIou`), loop for loop, on
bool masks.  TEST INFRASTRUCTURE ONLY.

*** PARITY UNPINNED ***  pycocotools is not vendored or installed; this restates its published
code.  Inputs are plain lists instead of COCO objects:

    gts: dicts {"image_id", "category_id", "mask" (bool [H, W]), "iscrowd", "area"}
    dts: dicts {"image_id", "category_id", "mask", "score"}, in results order

A detection's area is its mask's pixel count (what `loadRes` stores).  The one stated difference:
matches are recorded as positions (gt index, dt index) and tested against -1, where pycocotools
stores annotation ids and tests them for truth (an annotation with id 0 counts as unmatched there).
"""
from collections import defaultdict

import numpy as np


class Params:
    def __init__(self):
        self.imgIds = []
        self.catIds = []
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [1, 10, 100]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ["all", "small", "medium", "large"]
        self.useCats = 1


def rle_iou(d, g, iscrowd):
    """maskApi.c rleIou for one pair of bool masks."""
    i = int(np.count_nonzero(d & g))
    if i == 0:
        return 0.0
    u = int(np.count_nonzero(d)) if iscrowd else int(np.count_nonzero(d | g))
    return float(i) / float(u)


class COCOevalOracle:
    def __init__(self, gts, dts, params=None):
        self.params = params or Params()
        if not self.params.imgIds:
            self.params.imgIds = sorted({g["image_id"] for g in gts} | {d["image_id"] for d in dts})
        if not self.params.catIds:
            self.params.catIds = sorted({g["category_id"] for g in gts})
        self.gts_in, self.dts_in = gts, dts

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
                d = dict(d, id=did, iscrowd=0, area=int(np.count_nonzero(d["mask"])))
                self._dts[d["image_id"], d["category_id"]].append(d)

    def evaluate(self):
        p = self.params
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        p.maxDets = sorted(p.maxDets)
        self._prepare()
        self.ious = {(imgId, catId): self.computeIoU(imgId, catId)
                     for imgId in p.imgIds for catId in p.catIds}
        maxDet = p.maxDets[-1]
        self.evalImgs = [self.evaluateImg(imgId, catId, areaRng, maxDet)
                         for catId in p.catIds for areaRng in p.areaRng for imgId in p.imgIds]

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
        ious = np.zeros((len(dt), len(gt)))
        for di, d in enumerate(dt):
            for gi, g in enumerate(gt):
                ious[di, gi] = rle_iou(d["mask"], g["mask"], int(g["iscrowd"]))
        return ious

    def evaluateImg(self, imgId, catId, aRng, maxDet):
        p = self.params
        gt = self._gts[imgId, catId]
        dt = self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            g["_ignore"] = 1 if (g["ignore"] or (g["area"] < aRng[0] or g["area"] > aRng[1])) else 0
        gtind = np.argsort([g["_ignore"] for g in gt], kind="mergesort")
        gt = [gt[i] for i in gtind]
        dtind = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in dtind[0:maxDet]]
        iscrowd = [int(o["iscrowd"]) for o in gt]
        ious = (self.ious[imgId, catId][:, gtind] if len(self.ious[imgId, catId]) > 0
                else self.ious[imgId, catId])
        T = len(p.iouThrs)
        G = len(gt)
        D = len(dt)
        gtm = -np.ones((T, G), dtype=np.int64)
        dtm = -np.ones((T, D), dtype=np.int64)
        gtIg = np.array([g["_ignore"] for g in gt])
        dtIg = np.zeros((T, D))
        if not len(ious) == 0:
            for tind, t in enumerate(p.iouThrs):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > -1 and not iscrowd[gind]:
                            continue
                        if m > -1 and gtIg[m] == 0 and gtIg[gind] == 1:
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou = ious[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gtIg[m]
                    dtm[tind, dind] = m
                    gtm[tind, m] = dind
        a = np.array([d["area"] < aRng[0] or d["area"] > aRng[1] for d in dt]).reshape((1, len(dt)))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == -1, np.repeat(a, T, 0)))
        return {
            "image_id": imgId, "category_id": catId, "aRng": aRng, "maxDet": maxDet,
            "dtIds": [d["id"] for d in dt], "gtIds": [g["id"] for g in gt],
            # the matched gt by its position in the caller's gts list
            "dtMatchIds": (np.where(dtm > -1, np.array([g["id"] for g in gt])[np.maximum(dtm, 0)],
                                    -1) if G else dtm),
            "dtMatches": dtm, "gtMatches": gtm, "dtScores": [d["score"] for d in dt],
            "gtIgnore": gtIg, "dtIgnore": dtIg,
        }

    def accumulate(self):
        p = self.params
        T = len(p.iouThrs)
        R = len(p.recThrs)
        K = len(p.catIds)
        A = len(p.areaRng)
        M = len(p.maxDets)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        scores = -np.ones((T, R, K, A, M))
        I0 = len(p.imgIds)
        A0 = len(p.areaRng)
        for k in range(K):
            Nk = k * A0 * I0
            for a in range(A):
                Na = a * I0
                for m, maxDet in enumerate(p.maxDets):
                    E = [self.evalImgs[Nk + Na + i] for i in range(I0)]
                    E = [e for e in E if e is not None]
                    if len(E) == 0:
                        continue
                    dtScores = np.concatenate([e["dtScores"][0:maxDet] for e in E])
                    inds = np.argsort(-dtScores, kind="mergesort")
                    dtScoresSorted = dtScores[inds]
                    dtm = np.concatenate([e["dtMatches"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    dtIg = np.concatenate([e["dtIgnore"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    gtIg = np.concatenate([e["gtIgnore"] for e in E])
                    npig = np.count_nonzero(gtIg == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm > -1, np.logical_not(dtIg))
                    fps = np.logical_and(np.logical_not(dtm > -1), np.logical_not(dtIg))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        tp = np.array(tp)
                        fp = np.array(fp)
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q = np.zeros((R,))
                        ss = np.zeros((R,))
                        if nd:
                            recall[t, k, a, m] = rc[-1]
                        else:
                            recall[t, k, a, m] = 0
                        pr = pr.tolist()
                        q = q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        inds = np.searchsorted(rc, p.recThrs, side="left")
                        try:
                            for ri, pi in enumerate(inds):
                                q[ri] = pr[pi]
                                ss[ri] = dtScoresSorted[pi]
                        except IndexError:
                            pass
                        precision[t, :, k, a, m] = np.array(q)
                        scores[t, :, k, a, m] = np.array(ss)
        self.eval = {"params": p, "counts": [T, R, K, A, M], "precision": precision,
                     "recall": recall, "scores": scores}

    def summarize(self):
        def _summarize(ap=1, iouThr=None, areaRng="all", maxDets=100):
            p = self.params
            iStr = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}"
            titleStr = "Average Precision" if ap == 1 else "Average Recall"
            typeStr = "(AP)" if ap == 1 else "(AR)"
            iouStr = "{:0.2f}:{:0.2f}".format(p.iouThrs[0], p.iouThrs[-1]) \
                if iouThr is None else "{:0.2f}".format(iouThr)
            aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
            if ap == 1:
                s = self.eval["precision"]
                if iouThr is not None:
                    t = np.where(iouThr == p.iouThrs)[0]
                    s = s[t]
                s = s[:, :, :, aind, mind]
            else:
                s = self.eval["recall"]
                if iouThr is not None:
                    t = np.where(iouThr == p.iouThrs)[0]
                    s = s[t]
                s = s[:, :, aind, mind]
            if len(s[s > -1]) == 0:
                mean_s = -1
            else:
                mean_s = np.mean(s[s > -1])
            print(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
            return mean_s

        stats = np.zeros((12,))
        stats[0] = _summarize(1)
        stats[1] = _summarize(1, iouThr=.5, maxDets=self.params.maxDets[2])
        stats[2] = _summarize(1, iouThr=.75, maxDets=self.params.maxDets[2])
        stats[3] = _summarize(1, areaRng="small", maxDets=self.params.maxDets[2])
        stats[4] = _summarize(1, areaRng="medium", maxDets=self.params.maxDets[2])
        stats[5] = _summarize(1, areaRng="large", maxDets=self.params.maxDets[2])
        stats[6] = _summarize(0, maxDets=self.params.maxDets[0])
        stats[7] = _summarize(0, maxDets=self.params.maxDets[1])
        stats[8] = _summarize(0, maxDets=self.params.maxDets[2])
        stats[9] = _summarize(0, areaRng="small", maxDets=self.params.maxDets[2])
        stats[10] = _summarize(0, areaRng="medium", maxDets=self.params.maxDets[2])
        stats[11] = _summarize(0, areaRng="large", maxDets=self.params.maxDets[2])
        self.stats = stats
