#!/usr/bin/env python
"""Do the pre-processing tests notice a subtly wrong kernel?  Fourteen mutants of csrc/mold.cu and
csrc/anchors.cu, each one textual edit that computes wrong VALUES only (no mutant indexes out
of bounds), run by tools/mutants.py under the new test files and the older one:

    python tools/mutate_preprocess.py             # on a machine with the GPU
    python tools/mutate_preprocess.py --dry-run   # apply every edit and compile it, no tests
"""
import sys

import mutants

RESIZE, MOLD, ANCHORS = ("tests/test_gpu_cv2_resize.py", "tests/test_gpu_mold.py",
                         "tests/test_gpu_anchors.py")
NEW_TESTS = [RESIZE, MOLD, ANCHORS]
OLD_TESTS = ["tests/test_gpu_anchors_mold.py"]
# the 2.19 GB sources need 4.3 GB of device memory and no mutant needs them
DESELECT = ["tests/test_gpu_cv2_resize.py::test_source_past_2g_bytes"]
EQUIVALENT = set()


def first(test):
    """(new, old) selections with the file that tests the mutated kernel first, since each run
    stops at its first failure."""
    return [test] + [t for t in NEW_TESTS if t != test], OLD_TESTS


# the old file's batches do not start with their smallest image
BATCH_NEW = (["tests/test_gpu_cv2_resize.py::test_batch_equals_single",
              "tests/test_gpu_mold.py::test_preprocess_input_batch"], None)

ZOOM_SUM = """\
          double t = __dmul_rn(__dmul_rn(c00, zy.w0), zx.w0);
          t = __dadd_rn(t, __dmul_rn(__dmul_rn(c01, zy.w0), zx.w1));
          t = __dadd_rn(t, __dmul_rn(__dmul_rn(c10, zy.w1), zx.w0));
          t = __dadd_rn(t, __dmul_rn(__dmul_rn(c11, zy.w1), zx.w1));
"""
ZOOM_SUM_PAIRWISE = """\
          const double p00 = __dmul_rn(__dmul_rn(c00, zy.w0), zx.w0);
          const double p01 = __dmul_rn(__dmul_rn(c01, zy.w0), zx.w1);
          const double p10 = __dmul_rn(__dmul_rn(c10, zy.w1), zx.w0);
          const double p11 = __dmul_rn(__dmul_rn(c11, zy.w1), zx.w1);
          const double t = __dadd_rn(__dadd_rn(p00, p01), __dadd_rn(p10, p11));
"""
AREA_LOADS = """\
      const unsigned char *p0 = src + (static_cast<size_t>(2 * dy) * sw + 2 * dx) * 3;
      const unsigned char *p1 = p0 + static_cast<size_t>(sw) * 3;
"""
# the clamps of the linear branch, so that a 2x2 box on an axis that is not 2x stays in the source
AREA_LOADS_CLAMPED = """\
      const int ay0 = min(2 * dy, sh - 1), ay1 = min(2 * dy + 1, sh - 1);
      const int ax0 = min(2 * dx, sw - 1), ax1 = min(2 * dx + 1, sw - 1);
      const unsigned char *p0 = src + (static_cast<size_t>(ay0) * sw + ax0) * 3;
      const unsigned char *p1 = src + (static_cast<size_t>(ay1) * sw + ax0) * 3;
      const int ax = (ax1 - ax0) * 3;
"""
ANCHOR_DECODE = """\
    const int r = static_cast<int>(local % p.n_ratios);
    const long long cell = local / p.n_ratios;
    const int x = static_cast<int>(cell % p.nx[l]);
    const int y = static_cast<int>(cell / p.nx[l]);
"""
ANCHOR_DECODE_SWAPPED = """\
    const int x = static_cast<int>(local % p.nx[l]);
    const long long cell = local / p.nx[l];
    const int r = static_cast<int>(cell % p.n_ratios);
    const int y = static_cast<int>(cell / p.n_ratios);
"""

M, A = "mold.cu", "anchors.cu"
# (number, what it models, [(file, old, new, occurrences)], (new, old) selections)
MUTANTS = [
    (1, "mold: one multiply-add contracted into an FMA", [
        (M, "t = __dadd_rn(t, __dmul_rn(__dmul_rn(c11, zy.w1), zx.w1));",
         "t = fma(__dmul_rn(c11, zy.w1), zx.w1, t);", 1)], first(MOLD)),
    (2, "mold: the four products summed pairwise", [
        (M, ZOOM_SUM, ZOOM_SUM_PAIRWISE, 1)], first(MOLD)),
    (3, "mold: the source coordinate from one FMA", [
        (M, "__dsub_rn(__dmul_rn(static_cast<double>(k) + 0.5, zoom), 0.5);",
         "fma(static_cast<double>(k) + 0.5, zoom, -0.5);", 1)], first(MOLD)),
    (4, "mold: uint8 by rounding instead of truncation", [
        (M, "static_cast<unsigned char>(static_cast<int>(t));",
         "static_cast<unsigned char>(__double2int_rn(t));", 1)], first(MOLD)),
    (5, "mold: float32 output as float(px) - float(mean)", [
        (M, "out[i * 3 + c] = static_cast<TOut>(v);",
         "out[i * 3 + c] = sizeof(TOut) == 4 ? static_cast<TOut>(__fsub_rn("
         "static_cast<float>(px[c]), static_cast<float>(mean[c]))) : static_cast<TOut>(v);", 1)],
     first(MOLD)),
    # the loop bound is kept: later trips visit other pixels, none outside the image
    (6, "mold and resize: grid stride off by one", [
        (M, "i += static_cast<long long>(gridDim.x) * kMoldThreads)",
         "i += static_cast<long long>(gridDim.x) * kMoldThreads + 1)", 2)], first(RESIZE)),
    (7, "resize: area shortcut when either axis is 2x", [
        (M, "fabs(scale_x - 2.0) < eps && fabs(scale_y - 2.0) < eps;",
         "fabs(scale_x - 2.0) < eps || fabs(scale_y - 2.0) < eps;", 1),
        (M, AREA_LOADS, AREA_LOADS_CLAMPED, 1),
        (M, "(p0[c] + p0[3 + c] + p1[c] + p1[3 + c] + 2) >> 2",
         "(p0[c] + p0[ax + c] + p1[c] + p1[ax + c] + 2) >> 2", 1)], first(RESIZE)),
    (8, "resize: coefficients truncated, not cvRound", [
        (M, "= __float2int_rn(__fmul_rn(", "= __float2int_rz(__fmul_rn(", 2)], first(RESIZE)),
    (9, "resize: coordinate kept in double", [
        (M, "  float f = __double2float_rn(__dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, "
         "scale), 0.5));\n  int s = __float2int_rd(f);\n"
         "  f = __fsub_rn(f, static_cast<float>(s));\n",
         "  const double fd = __dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), 0.5);\n"
         "  int s = __double2int_rd(fd);\n"
         "  float f = __double2float_rn(__dsub_rn(fd, static_cast<double>(s)));\n", 1)],
     first(RESIZE)),
    (10, "resize: y weights clamped like x weights", [
        (M, "cv_lin_coef(dy, scale_y, sh, false);", "cv_lin_coef(dy, scale_y, sh, true);", 1)],
     first(RESIZE)),
    (11, "resize: vertical pass rounds with + 1", [
        (M, "((cy.a1 * (S1 >> 4)) >> 16) + 2) >> 2;", "((cy.a1 * (S1 >> 4)) >> 16) + 1) >> 2;", 1)],
     first(RESIZE)),
    # every image read with the sizes of image 0: run only on batches whose image 0 is the
    # smallest, so that every read stays inside its own slot
    (12, "resize batch: sizes of image 0 for every image", [
        (M, "sh = src_hw[2 * b];", "sh = src_hw[0];", 1),
        (M, "sw = src_hw[2 * b + 1];", "sw = src_hw[1];", 1)], BATCH_NEW),
    # (halving as a multiply is exact, so 0.5 * h as an FMA operand would be an equivalent mutant)
    # The reciprocal moves the float64 quotient by at most one ulp, which changes the float32
    # only for a quotient on a float32 rounding tie: about one value in 2^29, so no sweep meets
    # one; test_gpu_anchors.py::test_division_not_reciprocal constructs such scales.
    (13, "anchors: multiply by the reciprocal instead of dividing", [
        (A, "__ddiv_rn(y1, hm1)", "__dmul_rn(y1, __ddiv_rn(1.0, hm1))", 1),
        (A, "__ddiv_rn(x1, wm1)", "__dmul_rn(x1, __ddiv_rn(1.0, wm1))", 1),
        (A, "__ddiv_rn(__dsub_rn(y2, 1.0), hm1)",
         "__dmul_rn(__dsub_rn(y2, 1.0), __ddiv_rn(1.0, hm1))", 1),
        (A, "__ddiv_rn(__dsub_rn(x2, 1.0), wm1)",
         "__dmul_rn(__dsub_rn(x2, 1.0), __ddiv_rn(1.0, wm1))", 1)], first(ANCHORS)),
    (14, "anchors: ratio and x swapped in the row decode", [
        (A, ANCHOR_DECODE, ANCHOR_DECODE_SWAPPED, 1)], first(ANCHORS)),
]


if __name__ == "__main__":
    mutants.main(sys.modules[__name__])
