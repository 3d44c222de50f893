"""CPU restatement of lvis-api's evaluation (`LVISResults.limit_dets_per_image`; `LVISEval`:
`_prepare`, `compute_iou`, `evaluate_img`, `accumulate`, `summarize`, `print_results`;
`_prepare_freq_group`), loop for loop, on bool masks ("segm") or [x, y, w, h] boxes ("bbox").
TEST INFRASTRUCTURE ONLY.

*** PARITY UNPINNED ***  lvis-api is not vendored or installed; this restates its published code.
Inputs are plain lists instead of LVIS objects:

    gts: dicts {"image_id", "category_id", "mask" (bool [H, W]) or "bbox", "area"} ("iscrowd" may
         be present and is not read, as LVISEval does not read it)
    dts: dicts {"image_id", "category_id", "mask" or "bbox", "score"}, in results order
    images: dicts {"id", "neg_category_ids", "not_exhaustive_category_ids"}
    categories: dicts {"id", "frequency"}

A segm detection's area is its mask's pixel count, a bbox detection's w*h.  Stated differences:
matches are recorded as positions and tested against -1, where lvis-api stores annotation ids
and tests them for truth; NaN scores sort after every number in the per-image cut (Python's
`sorted` leaves their place undefined); there are no `dt_pointers`.
"""
from collections import OrderedDict, defaultdict

import numpy as np

from bbox_cocoeval_oracle import bb_iou
from cocoeval_oracle import rle_iou


class Params:
    def __init__(self, iou_type="segm"):
        self.img_ids = []
        self.cat_ids = []
        self.iou_thrs = np.linspace(0.5, 0.95, int(np.round((0.95 - 0.5) / 0.05)) + 1,
                                    endpoint=True)
        self.rec_thrs = np.linspace(0.0, 1.00, int(np.round((1.00 - 0.0) / 0.01)) + 1,
                                    endpoint=True)
        self.max_dets = 300
        self.area_rng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2],
                         [96 ** 2, 1e5 ** 2]]
        self.area_rng_lbl = ["all", "small", "medium", "large"]
        self.use_cats = 1
        self.img_count_lbl = ["r", "c", "f"]
        self.iou_type = iou_type


def limit_dets_per_image(dts, max_dets):
    """LVISResults.limit_dets_per_image: per image, the first max_dets of the results sorted by
    descending score (stable: equal scores keep results order; NaN last).  Returns the kept
    results, each with "id" its position in dts."""
    img_ann = defaultdict(list)
    for did, d in enumerate(dts):
        img_ann[d["image_id"]].append(dict(d, id=did))
    for img_id, anns in img_ann.items():
        if len(anns) <= max_dets:
            continue
        anns = sorted(anns, key=lambda a: (np.isnan(a["score"]), -a["score"]
                                           if not np.isnan(a["score"]) else 0.0))
        img_ann[img_id] = anns[:max_dets]
    return [a for anns in img_ann.values() for a in anns]


class LVISEvalOracle:
    def __init__(self, gts, dts, images, categories, iou_type="segm", params=None):
        self.params = params or Params(iou_type)
        self.params.iou_type = iou_type
        if not self.params.img_ids:
            self.params.img_ids = sorted(im["id"] for im in images)
        if not self.params.cat_ids:
            self.params.cat_ids = sorted(c["id"] for c in categories)
        self.images = {im["id"]: im for im in images}
        self.cats = {c["id"]: c for c in categories}
        self.gts_in = gts
        self.dts_in = limit_dets_per_image(dts, self.params.max_dets)
        self.results = OrderedDict()

    def _area(self, d):
        if self.params.iou_type == "segm":
            return int(np.count_nonzero(d["mask"]))
        bb = d["bbox"]
        return bb[2] * bb[3]

    def _prepare(self):
        p = self.params
        self._gts = defaultdict(list)
        self._dts = defaultdict(list)
        gts = [dict(g, id=gid) for gid, g in enumerate(self.gts_in)
               if g["image_id"] in p.img_ids and g["category_id"] in p.cat_ids]
        for g in gts:
            if "ignore" not in g:
                g["ignore"] = 0
        for g in gts:
            self._gts[g["image_id"], g["category_id"]].append(g)
        img_nl = {i: self.images[i]["neg_category_ids"] for i in p.img_ids}
        img_pl = defaultdict(set)
        for g in gts:
            img_pl[g["image_id"]].add(g["category_id"])
        self.img_nel = {i: self.images[i]["not_exhaustive_category_ids"] for i in p.img_ids}
        for d in self.dts_in:
            if d["image_id"] not in p.img_ids or d["category_id"] not in p.cat_ids:
                continue
            img_id, cat_id = d["image_id"], d["category_id"]
            if cat_id not in img_nl[img_id] and cat_id not in img_pl[img_id]:
                continue
            self._dts[img_id, cat_id].append(dict(d, area=self._area(d)))
        self.freq_groups = self._prepare_freq_group()

    def _prepare_freq_group(self):
        p = self.params
        freq_groups = [[] for _ in p.img_count_lbl]
        for idx, c in enumerate(p.cat_ids):
            freq_groups[p.img_count_lbl.index(self.cats[c]["frequency"])].append(idx)
        return freq_groups

    def evaluate(self):
        p = self.params
        p.img_ids = list(np.unique(p.img_ids))
        self._prepare()
        self.ious = {(i, c): self.compute_iou(i, c) for i in p.img_ids for c in p.cat_ids}
        self.eval_imgs = [self.evaluate_img(i, c, a) for c in p.cat_ids for a in p.area_rng
                          for i in p.img_ids]

    def compute_iou(self, img_id, cat_id):
        gt, dt = self._gts[img_id, cat_id], self._dts[img_id, cat_id]
        if len(gt) == 0 and len(dt) == 0:
            return []
        idx = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in idx]
        iscrowd = [0] * len(gt)
        if len(gt) == 0 or len(dt) == 0:       # mask_utils.iou of an empty side: []
            return []
        if self.params.iou_type == "segm":
            ious = np.zeros((len(dt), len(gt)))
            for di, d in enumerate(dt):
                for gi, g in enumerate(gt):
                    ious[di, gi] = rle_iou(d["mask"], g["mask"], iscrowd[gi])
            return ious
        return bb_iou([d["bbox"] for d in dt], [g["bbox"] for g in gt], iscrowd)

    def evaluate_img(self, img_id, cat_id, area_rng):
        gt, dt = self._gts[img_id, cat_id], self._dts[img_id, cat_id]
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            g["_ignore"] = 1 if (g["ignore"] or g["area"] < area_rng[0]
                                 or g["area"] > area_rng[1]) else 0
        gt_idx = np.argsort([g["_ignore"] for g in gt], kind="mergesort")
        gt = [gt[i] for i in gt_idx]
        dt_idx = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in dt_idx]
        ious = (self.ious[img_id, cat_id][:, gt_idx] if len(self.ious[img_id, cat_id]) > 0
                else self.ious[img_id, cat_id])
        T, G, D = len(self.params.iou_thrs), len(gt), len(dt)
        gt_m = -np.ones((T, G), np.int64)
        dt_m = -np.ones((T, D), np.int64)
        gt_ig = np.array([g["_ignore"] for g in gt])
        dt_ig = np.zeros((T, D))
        for t, thr in enumerate(self.params.iou_thrs):
            if len(ious) == 0:
                break
            for di, d in enumerate(dt):
                iou = min([thr, 1 - 1e-10])
                m = -1
                for gi, _ in enumerate(gt):
                    if gt_m[t, gi] > -1:
                        continue
                    if m > -1 and gt_ig[m] == 0 and gt_ig[gi] == 1:
                        break
                    if ious[di, gi] < iou:
                        continue
                    iou = ious[di, gi]
                    m = gi
                if m == -1:
                    continue
                dt_ig[t, di] = gt_ig[m]
                dt_m[t, di] = m
                gt_m[t, m] = di
        dt_ig_mask = np.array([d["area"] < area_rng[0] or d["area"] > area_rng[1]
                               or d["category_id"] in self.img_nel[d["image_id"]]
                               for d in dt]).reshape((1, D))
        dt_ig_mask = np.repeat(dt_ig_mask, T, 0)
        dt_ig = np.logical_or(dt_ig, np.logical_and(dt_m == -1, dt_ig_mask))
        return {
            "image_id": img_id, "category_id": cat_id, "area_rng": area_rng,
            "dt_ids": [d["id"] for d in dt], "gt_ids": [g["id"] for g in gt],
            # the matched gt by its position in the caller's gts list
            "dt_match_ids": (np.where(dt_m > -1, np.array([g["id"] for g in gt])[np.maximum(dt_m, 0)],
                                      -1) if G else dt_m),
            "dt_matches": dt_m, "gt_matches": gt_m, "dt_scores": [d["score"] for d in dt],
            "gt_ignore": gt_ig, "dt_ignore": dt_ig,
        }

    def accumulate(self):
        p = self.params
        T, R, K, A = len(p.iou_thrs), len(p.rec_thrs), len(p.cat_ids), len(p.area_rng)
        I0 = len(p.img_ids)
        precision = -np.ones((T, R, K, A))
        recall = -np.ones((T, K, A))
        for k in range(K):
            Nk = k * A * I0
            for a in range(A):
                Na = a * I0
                E = [self.eval_imgs[Nk + Na + i] for i in range(I0)]
                E = [e for e in E if e is not None]
                if len(E) == 0:
                    continue
                dt_scores = np.concatenate([e["dt_scores"] for e in E], axis=0)
                dt_idx = np.argsort(-dt_scores, kind="mergesort")
                dt_m = np.concatenate([e["dt_matches"] for e in E], axis=1)[:, dt_idx]
                dt_ig = np.concatenate([e["dt_ignore"] for e in E], axis=1)[:, dt_idx]
                gt_ig = np.concatenate([e["gt_ignore"] for e in E])
                num_gt = np.count_nonzero(gt_ig == 0)
                if num_gt == 0:
                    continue
                tps = np.logical_and(dt_m > -1, np.logical_not(dt_ig))
                fps = np.logical_and(np.logical_not(dt_m > -1), np.logical_not(dt_ig))
                tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                    tp = np.array(tp)
                    fp = np.array(fp)
                    num_tp = len(tp)
                    rc = tp / num_gt
                    if num_tp:
                        recall[t, k, a] = rc[-1]
                    else:
                        recall[t, k, a] = 0
                    pr = tp / (fp + tp + np.spacing(1))
                    pr = pr.tolist()
                    for i in range(num_tp - 1, 0, -1):
                        if pr[i] > pr[i - 1]:
                            pr[i - 1] = pr[i]
                    rec_thrs_insert_idx = np.searchsorted(rc, p.rec_thrs, side="left")
                    pr_at_recall = [0.0] * R
                    try:
                        for _idx, pr_idx in enumerate(rec_thrs_insert_idx):
                            pr_at_recall[_idx] = pr[pr_idx]
                    except IndexError:
                        pass
                    precision[t, :, k, a] = np.array(pr_at_recall)
        self.eval = {"params": p, "counts": [T, R, K, A], "precision": precision,
                     "recall": recall}

    def _summarize(self, summary_type, iou_thr=None, area_rng="all", freq_group_idx=None):
        p = self.params
        aidx = [idx for idx, lbl in enumerate(p.area_rng_lbl) if lbl == area_rng]
        if summary_type == "ap":
            s = self.eval["precision"]
            if iou_thr is not None:
                s = s[np.where(iou_thr == p.iou_thrs)[0]]
            if freq_group_idx is not None:
                s = s[:, :, self.freq_groups[freq_group_idx], aidx]
            else:
                s = s[:, :, :, aidx]
        else:
            s = self.eval["recall"]
            if iou_thr is not None:
                s = s[np.where(iou_thr == p.iou_thrs)[0]]
            s = s[:, :, aidx]
        if len(s[s > -1]) == 0:
            return -1
        return np.mean(s[s > -1])

    def summarize(self):
        max_dets = self.params.max_dets
        self.results["AP"] = self._summarize("ap")
        self.results["AP50"] = self._summarize("ap", iou_thr=0.50)
        self.results["AP75"] = self._summarize("ap", iou_thr=0.75)
        self.results["APs"] = self._summarize("ap", area_rng="small")
        self.results["APm"] = self._summarize("ap", area_rng="medium")
        self.results["APl"] = self._summarize("ap", area_rng="large")
        self.results["APr"] = self._summarize("ap", freq_group_idx=0)
        self.results["APc"] = self._summarize("ap", freq_group_idx=1)
        self.results["APf"] = self._summarize("ap", freq_group_idx=2)
        self.results["AR@{}".format(max_dets)] = self._summarize("ar")
        for area_rng in ["small", "medium", "large"]:
            key = "AR{}@{}".format(area_rng[0], max_dets)
            self.results[key] = self._summarize("ar", area_rng=area_rng)

    def print_results(self):
        template = (" {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} catIds={:>3s}] = "
                    "{:0.3f}")
        for key, value in self.results.items():
            max_dets = self.params.max_dets
            if "AP" in key:
                title = "Average Precision"
                _type = "(AP)"
            else:
                title = "Average Recall"
                _type = "(AR)"
            if len(key) > 2 and key[2].isdigit():
                iou_thr = (float(key[2:]) / 100)
                iou = "{:0.2f}".format(iou_thr)
            else:
                iou = "{:0.2f}:{:0.2f}".format(self.params.iou_thrs[0], self.params.iou_thrs[-1])
            if len(key) > 2 and key[2] in ["r", "c", "f"]:
                cat_group_name = key[2]
            else:
                cat_group_name = "all"
            if len(key) > 2 and key[2] in ["s", "m", "l"]:
                area_rng = key[2]
            else:
                area_rng = "all"
            print(template.format(title, _type, iou, area_rng, max_dets, cat_group_name, value))

    def run(self):
        self.evaluate()
        self.accumulate()
        self.summarize()
