#!/usr/bin/env python
"""Do the JPEG tests notice a decoder that is subtly wrong?  Value-only mutants of the decode
kernels (csrc/jpeg.cu), each put under the edge tests and the older JPEG tests:

    python tools/mutate_jpeg.py             # on a machine with the GPU
    python tools/mutate_jpeg.py --dry-run   # apply every edit and compile it, no tests

Each mutant is built as its own library through tools/mutate_eval.py's copy-and-build (build.py's
MRX_LIB_NAME hook) and selected with MRX_LIB.  Every edit changes a value, never an index or a
bound: the dropped run past 63 still stores to the guard entry's index, only the value changes.
The IDCT mutants are the one-mistake variants of tests/jpeg_oracle.py's idct_islow, ported to
the kernel.  The repository's sources and build are not touched.  A development script: no test
imports it."""
import argparse
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mutate_eval as ME  # noqa: E402
from mutate_polygons import apply, run_tests  # noqa: E402
from matterport_maskrcnn_with_tensorflow_serving_b200 import build as B  # noqa: E402

NEW_TESTS = ["tests/test_gpu_jpeg_edges.py"]
OLD_TESTS = ["tests/test_gpu_jpeg.py", "tests/test_gpu_jpeg_progressive.py"]

F = "jpeg.cu"
_PX = "px[k] = (unsigned char)(min(max((o[k] + (1 << (sh - 1))) >> sh, -128), 127) + 128);"
# (number, what it models, [(old, new, occurrences)])
MUTANTS = [
    (1, "c: pass 2 through jidctint.c's range-limit table at x & 1023", [
        (_PX, "{ const int t = ((o[k] + (1 << (sh - 1))) >> sh) & 1023;\n"
              "        px[k] = (unsigned char)(t < 128 ? t + 128 : t < 512 ? 255 : t < 896 ? 0 "
              ": t - 896); }", 1)]),
    (2, "unwrapped_product: dequantised value kept in 32 bits", [
        ("x[k] = short(v * short(q[k * 8 + r]));", "x[k] = v * short(q[k * 8 + r]);", 1)]),
    (3, "unsigned_quant: quantiser unsigned, product kept in 32 bits", [
        ("x[k] = short(v * short(q[k * 8 + r]));", "x[k] = v * q[k * 8 + r];", 1)]),
    (4, "wide_sums: in0 +- in4 in 32 bits", [
        ("int(short(x[0] + x[4]))", "(x[0] + x[4])", 1),
        ("int(short(x[0] - x[4]))", "(x[0] - x[4])", 1)]),
    (5, "wide_sums: in7 + in3 and in5 + in1 in 32 bits", [
        ("const int z3 = short(x[7] + x[3]), z4 = short(x[5] + x[1]);",
         "const int z3 = x[7] + x[3], z4 = x[5] + x[1];", 1)]),
    (6, "pass1_wraps: pass-1 results wrapped to int16, not saturated", [
        ("w[k * 8 + r] = short(sat16((o[k] + half) >> (CONST_BITS - PASS1_BITS)));",
         "w[k * 8 + r] = short((o[k] + half) >> (CONST_BITS - PASS1_BITS));", 1)]),
    (7, "shortcut_dequantised: the shortcut tested on dequantised coefficients", [
        ("if (k) ac |= v != 0;", "if (k) ac |= x[k] != 0;", 1)]),
    (8, "shortcut_saturates: the shortcut's << 2 saturating", [
        ("const short v = short(x[0] * (1 << PASS1_BITS));",
         "const short v = short(sat16(x[0] * (1 << PASS1_BITS)));", 1)]),
    (9, "h2v1 rounding: + 2 for both phases", [
        ("return (3 * row[j] + row[jn] + 1 + odd) >> 2;", "return (3 * row[j] + row[jn] + 2) >> 2;",
         1)]),
    (10, "h2v2 rounding: + 7 + odd for 8 - odd", [
        ("return (3 * cs + cn + 8 - odd) >> 4;", "return (3 * cs + cn + 7 + odd) >> 4;", 1)]),
    (11, "narrow chroma: fancy upsampling from 2 samples wide", [
        ("if (he == 2 && dw > 2 && (ve == 1 || ve == 2))",
         "if (he == 2 && dw > 1 && (ve == 1 || ve == 2))", 1)]),
    (12, "colour table without the + 0.5 of FIX(x)", [
        ("-46802 * cr + (-22554 * cb", "-46801 * cr + (-22553 * cb", 1),
        ("116130 * cb", "116129 * cb", 1)]),
    (13, "DC stored saturated to int16, not truncated", [
        ("*q = short(int(v));", "*q = short(max(-32768LL, min(v, 32767LL)));", 1)]),
    (14, "a run past 63 dropped (its guard entry's store writes 0)", [
        ("if (kWrite) coef[size_t(cur) * 64 + c_zigzag[z]] = short(v);",
         "if (kWrite) coef[size_t(cur) * 64 + c_zigzag[z]] = short(z > 63 ? 0 : v);", 1)]),
]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--dry-run", action="store_true", help="edit and compile only")
    ap.add_argument("--only", type=int, nargs="*", help="mutant numbers (default: all)")
    ap.add_argument("--logs", help="directory for each run's pytest output")
    ap.add_argument("--new-only", action="store_true", help="run only the new tests")
    ap.add_argument("--old-only", action="store_true", help="run only the older tests")
    args = ap.parse_args()
    if args.logs:
        os.makedirs(args.logs, exist_ok=True)
    B.build()     # the real library, whose objects the mutants share
    rows = []
    for number, what, edits in MUTANTS:
        if args.only and number not in args.only:
            continue
        tmp = tempfile.mkdtemp(prefix="mrx_jpeg_mutant_")
        try:
            csrc = ME.mutate(tmp, [])
            apply(os.path.join(csrc, F), [(F,) + e for e in edits])
            assert os.path.exists(ME.build_mutant(number, csrc))
            env = {"MRX_LIB": f"libmrx_mutant{number}.so"}
            if args.dry_run:
                row = (number, what, "built", "built")
            else:
                row = (number, what,
                       "not run" if args.old_only else
                       run_tests(NEW_TESTS, ROOT, env, "new", number, args.logs),
                       "not run" if args.new_only else
                       run_tests(OLD_TESTS, ROOT, env, "old", number, args.logs))
            rows.append(row)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
            ME.remove_mutant(number)
        print("| {} | {} | {} | {} |".format(*rows[-1]), flush=True)
    print("\n| # | mutant | new tests | old tests |\n|---|---|---|---|")
    for row in rows:
        print("| {} | {} | {} | {} |".format(*row))
    survivors = [r[0] for r in rows if r[2] == "survived"]
    if survivors:
        raise SystemExit(f"the new tests let mutants {survivors} live")


if __name__ == "__main__":
    main()
