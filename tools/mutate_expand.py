#!/usr/bin/env python
"""Do the mask-expand tests notice a kernel that is off by an ulp?  Ten mutants of the expand
kernels (csrc/expand.cuh, expand_team.cu, unmold.cu, expand_bits.cu, rle.cu), each a textual
edit that changes VALUES only (no mutant indexes out of bounds; none touches the NaN threshold
of the columns outside a box), run by tools/mutants.py under the new test file and the older
ones:

    python tools/mutate_expand.py             # on a machine with the GPU
    python tools/mutate_expand.py --dry-run   # apply every edit and compile it, no tests
"""
import sys

import mutants

NEW_TESTS = ["tests/test_gpu_expand_exact.py"]
OLD_TESTS = ["tests/test_gpu_unmold.py", "tests/test_gpu_tile_shapes.py",
             "tests/test_gpu_kernel_paths.py", "tests/test_gpu_pack.py", "tests/test_gpu_rle.py"]
# the cases that need gigabytes of device memory (and minutes); no mutant needs them
DESELECT = ["tests/test_gpu_unmold.py::test_full_size_properties",
            "tests/test_gpu_unmold.py::test_config4_4k_shape_properties",
            "tests/test_gpu_unmold.py::test_exhaustive_config4_4k",
            "tests/test_gpu_rle.py::test_rle_full_size_batch"]
EQUIVALENT = set()

SRC_FLOOR = """\
  int rem = A - i * D;
  if (rem < 0) {
    --i;
    rem += D;
  } else if (rem >= D) {
    ++i;
    rem -= D;
  }
  return {i, rem};
"""
SRC_FLOOR_UNCORRECTED = """\
  int rem = A - i * D;
  return {i, rem};
"""

# (number, what it models, [(file, old, new, occurrences)])
MUTANTS = [
    (1, "team kernel: > 0.5 instead of >= 0.5", [
        ("expand_team.cu", "if (v >= thr)", "if (v > thr)", 1),
        ("expand_team.cu", "if (v >= 0.5f && colvalid)", "if (v > 0.5f && colvalid)", 1)]),
    (2, "generic kernel: > 0.5 instead of >= 0.5", [
        ("unmold.cu", "if (lerp(e.wy, ht, hb) >= 0.5f && off < ulen)",
         "if (lerp(e.wy, ht, hb) > 0.5f && off < ulen)", 1)]),
    (3, "packed kernel: > 0.5 instead of >= 0.5", [
        ("expand_bits.cu", "__ballot_sync(0xffffffffu, v >= thr[c])",
         "__ballot_sync(0xffffffffu, v > thr[c])", 1)]),
    (4, "RLE kernel: > 0.5 instead of >= 0.5", [
        ("rle.cu", "cur = v >= thr;", "cur = v > thr;", 1),
        ("rle.cu", "vl >= 0.5f;", "vl > 0.5f;", 1)]),
    (5, "every kernel: lerp as a multiply and an add", [
        ("expand.cuh", "return fmaf(w, hi - lo, lo);", "return __fadd_rn(__fmul_rn(w, hi - lo), lo);",
         1)]),
    (6, "team kernel: 1/D of the columns rounded toward zero", [
        ("expand_team.cu", "e.invD = __fdiv_rn(1.0f, static_cast<float>(2 * (bx.w - bx.y)));",
         "e.invD = __frcp_rz(static_cast<float>(2 * (bx.w - bx.y)));", 1)]),
    (7, "generic kernel: 1/D of the columns rounded toward zero", [
        ("unmold.cu", "e.invD = __fdiv_rn(1.0f, static_cast<float>(e.D));",
         "e.invD = __frcp_rz(static_cast<float>(e.D));", 1)]),
    (8, "packed kernel: 1/D of the columns rounded toward zero", [
        ("expand_bits.cu", "const float invD = __fdiv_rn(1.0f, static_cast<float>(D));",
         "const float invD = __frcp_rz(static_cast<float>(D));", 1)]),
    (9, "RLE kernel: 1/D of the columns rounded toward zero", [
        ("rle.cu", "const float invD = __fdiv_rn(1.0f, static_cast<float>(D));",
         "const float invD = __frcp_rz(static_cast<float>(D));", 1)]),
    # the estimate is never too high (test_expand_oracle.py): without the correction a too-low
    # floor keeps rem = D, weight ~1 on the row / column below, every index still in range
    (10, "every kernel: src_floor without its correction", [
        ("expand.cuh", SRC_FLOOR, SRC_FLOOR_UNCORRECTED, 1)]),
]


if __name__ == "__main__":
    mutants.main(sys.modules[__name__])
