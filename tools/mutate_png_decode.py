#!/usr/bin/env python
"""Do the PNG decode tests notice a decoder that is subtly wrong?  Value-only mutants of
csrc/png_decode.cu, run by tools/mutants.py under the edge tests and the older PNG decode tests:

    python tools/mutate_png_decode.py             # on a machine with the GPU
    python tools/mutate_png_decode.py --dry-run   # apply every edit and compile it, no tests

Every edit changes a value or a condition, never an index or a bound of a loop over memory."""
import sys

import mutants

NEW_TESTS = ["tests/test_gpu_png_edges.py"]
OLD_TESTS = ["tests/test_gpu_png_decode.py"]
DESELECT = []
EQUIVALENT = {10}     # no input tells it from the kernel: DESIGN.md §3.23

F = "png_decode.cu"
_SLOW = "for (int l = 1; l < 16; ++l) {\n    code |= int(br.buf & 1);"
# (number, what it models, [(file, old, new, occurrences)])
MUTANTS = [
    (1, "the slow path stops at 14 bits (l < 15): no 15-bit codes", [
        (F, _SLOW, _SLOW.replace("l < 16", "l < 15"), 1)]),
    (2, "huff_build refuses a single 1-bit code (codes || maxlen != 1 -> true)", [
        (F, "if (left > 0 && (codes || maxlen != 1) && ncodes > 0) return -2;",
         "if (left > 0 && true && ncodes > 0) return -2;", 1)]),
    (3, "huff_build refuses an empty distance code (codes && ncodes == 0 -> ncodes == 0)", [
        (F, "if (codes && ncodes == 0) return -2;", "if (ncodes == 0) return -2;", 1)]),
    (4, "the window bound at zlib's MAX_DIST (dist > wsize - 262)", [
        (F, "if (dist > wsize || (absolute && dist > p)) {",
         "if (dist > wsize - 262 || (absolute && dist > p)) {", 1)]),
    (5, "lengths of code 284 clamped to 257", [
        (F, "len = c_base_length[c] + 3 + int(br.get(c_extra_lbits[c]));",
         "len = min(c_base_length[c] + 3 + int(br.get(c_extra_lbits[c])), c == 27 ? 257 : 258);",
         1)]),
    (6, "a code-length repeat across HLIT refused as an overrun", [
        (F, "            if (have + rep > nlen + ndist) {",
         "            if (have + rep > nlen + ndist || (have < nlen && have + rep > nlen)) {", 1)]),
    # 7, the chain's `redo = r.need > p` -> false, is not built: the chain then lists a block
    # whose copy reaches before the stream, the expand stops at that copy's distance error and
    # leaves the rest of the block's cells unwritten, and the resolve reads them as references
    # (DESIGN.md §3.23 states which test it fails)
    (8, "the finder refuses a single 1-bit code (header_ok's maxl != 1 -> true)", [
        (F, "if (lf > 0 && nc > 0 && maxl != 1) return false;",
         "if (lf > 0 && nc > 0 && true) return false;", 1)]),
    (9, "stored alignment drops a whole byte when already aligned", [
        (F, "br.get(br.cnt & 7);", "br.get(br.cnt & 7 ? br.cnt & 7 : 8);", 1)]),
    (10, "Paeth prefers b when pa == pb (equivalent: pa == pb <= pc forces a == b)", [
        (F, "return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;",
         "return pa < pb && pa <= pc ? a : pb <= pc ? b : c;", 1)]),
    (11, "Paeth prefers c when pa == pc < pb", [
        (F, "return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;",
         "return pa <= pb && pa < pc ? a : pb <= pc ? b : c;", 1)]),
]


if __name__ == "__main__":
    mutants.main(sys.modules[__name__])
