#!/usr/bin/env python
"""Do the PNG decode tests notice a decoder that is subtly wrong?  Value-only mutants of
csrc/png_decode.cu, each put under the edge tests and the older PNG decode tests:

    python tools/mutate_png_decode.py             # on a machine with the GPU
    python tools/mutate_png_decode.py --dry-run   # apply every edit and compile it, no tests

Each mutant is built as its own library through tools/mutate_eval.py's copy-and-build (build.py's
MRX_LIB_NAME hook) and selected with MRX_LIB.  Every edit changes a value or a condition, never
an index or a bound of a loop over memory.  The repository's sources and build are not touched.
A development script: no test imports it."""
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

NEW_TESTS = ["tests/test_gpu_png_edges.py"]
OLD_TESTS = ["tests/test_gpu_png_decode.py"]

F = "png_decode.cu"
_SLOW = "for (int l = 1; l < 16; ++l) {\n    code |= int(br.buf & 1);"
# (number, what it models, [(old, new, occurrences)])
MUTANTS = [
    (1, "the slow path stops at 14 bits (l < 15): no 15-bit codes", [
        (_SLOW, _SLOW.replace("l < 16", "l < 15"), 1)]),
    (2, "huff_build refuses a single 1-bit code (codes || maxlen != 1 -> true)", [
        ("if (left > 0 && (codes || maxlen != 1) && ncodes > 0) return -2;",
         "if (left > 0 && true && ncodes > 0) return -2;", 1)]),
    (3, "huff_build refuses an empty distance code (codes && ncodes == 0 -> ncodes == 0)", [
        ("if (codes && ncodes == 0) return -2;", "if (ncodes == 0) return -2;", 1)]),
    (4, "the window bound at zlib's MAX_DIST (dist > wsize - 262)", [
        ("if (dist > wsize || (absolute && dist > p)) {",
         "if (dist > wsize - 262 || (absolute && dist > p)) {", 1)]),
    (5, "lengths of code 284 clamped to 257", [
        ("len = c_base_length[c] + 3 + int(br.get(c_extra_lbits[c]));",
         "len = min(c_base_length[c] + 3 + int(br.get(c_extra_lbits[c])), c == 27 ? 257 : 258);",
         1)]),
    (6, "a code-length repeat across HLIT refused as an overrun", [
        ("            if (have + rep > nlen + ndist) {",
         "            if (have + rep > nlen + ndist || (have < nlen && have + rep > nlen)) {", 1)]),
    # 7, the chain's `redo = r.need > p` -> false, is not built: the chain then lists a block
    # whose copy reaches before the stream, the expand stops at that copy's distance error and
    # leaves the rest of the block's cells unwritten, and the resolve reads them as references
    # (DESIGN.md §3.23 states which test it fails)
    (8, "the finder refuses a single 1-bit code (header_ok's maxl != 1 -> true)", [
        ("if (lf > 0 && nc > 0 && maxl != 1) return false;",
         "if (lf > 0 && nc > 0 && true) return false;", 1)]),
    (9, "stored alignment drops a whole byte when already aligned", [
        ("br.get(br.cnt & 7);", "br.get(br.cnt & 7 ? br.cnt & 7 : 8);", 1)]),
    (10, "Paeth prefers b when pa == pb (equivalent: pa == pb <= pc forces a == b)", [
        ("return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;",
         "return pa < pb && pa <= pc ? a : pb <= pc ? b : c;", 1)]),
    (11, "Paeth prefers c when pa == pc < pb", [
        ("return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;",
         "return pa <= pb && pa < pc ? a : pb <= pc ? b : c;", 1)]),
]

EQUIVALENT = {10}     # no input tells it from the kernel: DESIGN.md §3.23


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
        tmp = tempfile.mkdtemp(prefix="mrx_png_mutant_")
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
    survivors = [r[0] for r in rows if r[2] == "survived" and r[0] not in EQUIVALENT]
    if survivors:
        raise SystemExit(f"the new tests let mutants {survivors} live")


if __name__ == "__main__":
    main()
