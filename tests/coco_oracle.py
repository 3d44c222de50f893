"""CPU restatement of the COCO output side: pycocotools' compressed RLE strings and upstream's
`build_coco_results`.  TEST INFRASTRUCTURE ONLY.

*** PARITY UNPINNED ***  pycocotools is not installed here and Matterport's samples/coco/coco.py
is not vendored by the reference.  `rle_to_string` / `rle_from_string` restate the published
format (pycocotools maskApi.c rleToString / rleFrString); `build_coco_results` restates upstream's
loop over the oracle's `unmold_detections` output, with `oracle.rle_encode` + `rle_to_string` in
place of `maskUtils.encode`.
"""
import numpy as np

import oracle


def rle_to_string(counts):
    """[PUBLISHED FORMAT, pycocotools maskApi.c rleToString] the "counts" string of `mask.encode`
    for uncompressed run lengths: run i becomes x = cnts[i] - cnts[i-2] when i > 2 (cnts[i]
    otherwise), written 5 bits at a time, least significant first, as chr(48 + group), with 0x20
    added while more groups follow; the last group's bit 0x10 is the sign."""
    cnts = [int(c) for c in counts]
    out = bytearray()
    for i, x in enumerate(cnts):
        if i > 2:
            x -= cnts[i - 2]
        more = True
        while more:
            c = x & 0x1F
            x >>= 5
            more = x != -1 if c & 0x10 else x != 0
            if more:
                c |= 0x20
            out.append(c + 48)
    return bytes(out)


def rle_from_string(s):
    """[PUBLISHED FORMAT, pycocotools maskApi.c rleFrString] inverse of `rle_to_string`: list of
    int run lengths."""
    cnts = []
    p = 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1F) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and c & 0x10:
                x |= -1 << (5 * k)
        if len(cnts) > 2:
            x += cnts[-2]
        cnts.append(x)
    return cnts


def encode(mask):
    """What `pycocotools.mask.encode(np.asfortranarray(mask))` returns for one [H, W] mask."""
    rle = oracle.rle_encode(mask)
    return {"size": rle["size"], "counts": rle_to_string(rle["counts"])}


def build_coco_results(image_ids, rois, class_ids, scores, masks, category_ids=None):
    """[UPSTREAM samples/coco/coco.py build_coco_results] one result dict per detection per
    image id -- upstream repeats the one image's detections for every id in `image_ids`.
    `category_ids[class_id]` stands in for `dataset.get_source_class_id(class_id, "coco")`
    (None: the class id itself)."""
    if rois is None:
        return []
    results = []
    for image_id in image_ids:
        for i in range(rois.shape[0]):
            class_id = class_ids[i]
            score = scores[i]
            bbox = np.around(rois[i], 1)
            mask = masks[:, :, i]
            results.append({
                "image_id": image_id,
                "category_id": class_id if category_ids is None else category_ids[class_id],
                "bbox": [bbox[1], bbox[0], bbox[3] - bbox[1], bbox[2] - bbox[0]],
                "score": score,
                "segmentation": encode(np.asfortranarray(mask)),
            })
    return results
