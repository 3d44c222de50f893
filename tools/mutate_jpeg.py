#!/usr/bin/env python
"""Do the JPEG tests notice a decoder that is subtly wrong?  Value-only mutants of the decode
kernels (csrc/jpeg.cu), run by tools/mutants.py under the edge tests and the older JPEG tests:

    python tools/mutate_jpeg.py             # on a machine with the GPU
    python tools/mutate_jpeg.py --dry-run   # apply every edit and compile it, no tests

Every edit changes a value, never an index or a bound: the dropped run past 63 still stores to
the guard entry's index, only the value changes.  The IDCT mutants are the one-mistake variants
of tests/jpeg_oracle.py's idct_islow, ported to the kernel."""
import sys

import mutants

NEW_TESTS = ["tests/test_gpu_jpeg_edges.py"]
OLD_TESTS = ["tests/test_gpu_jpeg.py", "tests/test_gpu_jpeg_progressive.py"]
DESELECT = []
EQUIVALENT = set()

F = "jpeg.cu"
_PX = "px[k] = (unsigned char)(min(max((o[k] + (1 << (sh - 1))) >> sh, -128), 127) + 128);"
# (number, what it models, [(file, old, new, occurrences)])
MUTANTS = [
    (1, "c: pass 2 through jidctint.c's range-limit table at x & 1023", [
        (F, _PX, "{ const int t = ((o[k] + (1 << (sh - 1))) >> sh) & 1023;\n"
                 "        px[k] = (unsigned char)(t < 128 ? t + 128 : t < 512 ? 255 : t < 896 ? 0 "
                 ": t - 896); }", 1)]),
    (2, "unwrapped_product: dequantised value kept in 32 bits", [
        (F, "x[k] = short(v * short(q[k * 8 + r]));", "x[k] = v * short(q[k * 8 + r]);", 1)]),
    (3, "unsigned_quant: quantiser unsigned, product kept in 32 bits", [
        (F, "x[k] = short(v * short(q[k * 8 + r]));", "x[k] = v * q[k * 8 + r];", 1)]),
    (4, "wide_sums: in0 +- in4 in 32 bits", [
        (F, "int(short(x[0] + x[4]))", "(x[0] + x[4])", 1),
        (F, "int(short(x[0] - x[4]))", "(x[0] - x[4])", 1)]),
    (5, "wide_sums: in7 + in3 and in5 + in1 in 32 bits", [
        (F, "const int z3 = short(x[7] + x[3]), z4 = short(x[5] + x[1]);",
         "const int z3 = x[7] + x[3], z4 = x[5] + x[1];", 1)]),
    (6, "pass1_wraps: pass-1 results wrapped to int16, not saturated", [
        (F, "w[k * 8 + r] = short(sat16((o[k] + half) >> (CONST_BITS - PASS1_BITS)));",
         "w[k * 8 + r] = short((o[k] + half) >> (CONST_BITS - PASS1_BITS));", 1)]),
    (7, "shortcut_dequantised: the shortcut tested on dequantised coefficients", [
        (F, "if (k) ac |= v != 0;", "if (k) ac |= x[k] != 0;", 1)]),
    (8, "shortcut_saturates: the shortcut's << 2 saturating", [
        (F, "const short v = short(x[0] * (1 << PASS1_BITS));",
         "const short v = short(sat16(x[0] * (1 << PASS1_BITS)));", 1)]),
    (9, "h2v1 rounding: + 2 for both phases", [
        (F, "return (3 * row[j] + row[jn] + 1 + odd) >> 2;",
         "return (3 * row[j] + row[jn] + 2) >> 2;", 1)]),
    (10, "h2v2 rounding: + 7 + odd for 8 - odd", [
        (F, "return (3 * cs + cn + 8 - odd) >> 4;", "return (3 * cs + cn + 7 + odd) >> 4;", 1)]),
    (11, "narrow chroma: fancy upsampling from 2 samples wide", [
        (F, "if (he == 2 && dw > 2 && (ve == 1 || ve == 2))",
         "if (he == 2 && dw > 1 && (ve == 1 || ve == 2))", 1)]),
    (12, "colour table without the + 0.5 of FIX(x)", [
        (F, "-46802 * cr + (-22554 * cb", "-46801 * cr + (-22553 * cb", 1),
        (F, "116130 * cb", "116129 * cb", 1)]),
    (13, "DC stored saturated to int16, not truncated", [
        (F, "*q = short(int(v));", "*q = short(max(-32768LL, min(v, 32767LL)));", 1)]),
    (14, "a run past 63 dropped (its guard entry's store writes 0)", [
        (F, "if (kWrite) coef[size_t(cur) * 64 + c_zigzag[z]] = short(v);",
         "if (kWrite) coef[size_t(cur) * 64 + c_zigzag[z]] = short(z > 63 ? 0 : v);", 1)]),
]


if __name__ == "__main__":
    mutants.main(sys.modules[__name__])
