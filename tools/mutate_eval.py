#!/usr/bin/env python
"""Do the scoring tests notice a kernel that breaks a tie or a bound the other way?  Fifteen
mutants of the scoring kernels (csrc/cocoeval.cu, overlaps.cu, planes.cuh), each a textual edit
that changes VALUES only (no mutant indexes out of bounds), run by tools/mutants.py under the new
test file and the older ones:

    python tools/mutate_eval.py             # on a machine with the GPU
    python tools/mutate_eval.py --dry-run   # apply every edit and compile it, no tests
"""
import sys

import mutants

NEW_TESTS = ["tests/test_gpu_score_edges.py"]
OLD_TESTS = ["tests/test_gpu_cocoeval.py", "tests/test_gpu_cocoeval_bbox.py",
             "tests/test_gpu_cocoeval_boundary.py", "tests/test_gpu_eval.py",
             "tests/test_gpu_lvis.py"]
DESELECT = []
EQUIVALENT = set()

# (number, what it models, [(file, old, new, occurrences)])
MUTANTS = [
    (1, "coco_match: lane ties to the smaller j (key > best)", [
        ("cocoeval.cu", "if (key >= best || bj < 0)", "if (key > best || bj < 0)", 1)]),
    (2, "coco_match: ties across lanes to the smaller j (oj < bj)", [
        ("cocoeval.cu", "(ok == best && oj > bj)", "(ok == best && oj < bj)", 1)]),
    (3, "coco_match: strict IoU threshold (v > thr)", [
        ("cocoeval.cu", "if (!(v >= thr)) continue;", "if (!(v > thr)) continue;", 1)]),
    (4, "coco_match: ground truth at the lower area bound ignored (ga <= lo)", [
        ("cocoeval.cu", "crowd || ga < lo || ga > hi", "crowd || ga <= lo || ga > hi", 1)]),
    (5, "coco_match: unmatched detection at the upper bound ignored (da >= hi)", [
        ("cocoeval.cu", "ig = da < lo || da > hi;", "ig = da < lo || da >= hi;", 1)]),
    (6, "coco_match: crowd instances matched only once", [
        ("cocoeval.cu", "if (!crowd && (s_matched[j >> 5] >> (j & 31) & 1u)) continue;",
         "if ((s_matched[j >> 5] >> (j & 31) & 1u)) continue;", 1)]),
    (7, "mask_match: NaN keyed as IoU 0, below every number", [
        ("overlaps.cu", "key = (2ull << 62) | static_cast<unsigned>(j);",
         "key = (1ull << 62) | static_cast<unsigned>(j);", 1)]),
    (8, "mask_match: strict IoU threshold (> thr)", [
        ("overlaps.cu", "static_cast<double>(v) >= thr &&", "static_cast<double>(v) > thr &&", 1)]),
    (9, "mask_match: IoU ties to the smaller j", [
        ("overlaps.cu", "static_cast<unsigned>(j);", "(0xFFFFu - static_cast<unsigned>(j));", 2),
        ("overlaps.cu", "static_cast<int>(best & 0xFFFFu)",
         "static_cast<int>(0xFFFFu - (best & 0xFFFFu))", 1)]),
    (10, "mask_rank: score ties to the smaller index (k < i)", [
        ("overlaps.cu", "(tie && k > i)", "(tie && k < i)", 1)]),
    (11, "rle_iou: crowd union from the ground truth's area (a2)", [
        ("cocoeval.cu", "const long long u = crowd ? a1 : a1 + a2 - inter;",
         "const long long u = crowd ? a2 : a1 + a2 - inter;", 1)]),
    (12, "and_count: first-byte mask from (x1 + 1) & 7", [
        ("planes.cuh", "first = 0xFFu >> (x1 & 7)", "first = 0xFFu >> ((x1 + 1) & 7)", 1)]),
    (13, "and_count: last-byte mask shifted by one", [
        ("planes.cuh", "last = (0xFFu << (7 - ((x2 - 1) & 7))) & 0xFFu",
         "last = (0xFFu << (8 - ((x2 - 1) & 7))) & 0xFFu", 1)]),
    (14, "coco_box_iou: da + g[2]*g[3] contracted into an fma", [
        ("cocoeval.cu", "__dsub_rn(__dadd_rn(da, __dmul_rn(g[2], g[3])), inter)",
         "__dsub_rn(__fma_rn(g[2], g[3], da), inter)", 1)]),
    (15, "LVIS keep: the cut by rank in the category instead of the walk", [
        ("cocoeval.cu", "int b, int ci, int,", "int b, int ci, int rank,", 1),
        ("cocoeval.cu", "walk < p.max_det &&", "rank < p.max_det &&", 1)]),
]


if __name__ == "__main__":
    mutants.main(sys.modules[__name__])
