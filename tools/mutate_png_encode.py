#!/usr/bin/env python
"""Do the PNG encode tests notice an encoder that is subtly wrong?  Value-only mutants of
csrc/png.cu, run by tools/mutants.py under the edge tests and the older PNG encode tests:

    python tools/mutate_png_encode.py             # on a machine with the GPU
    python tools/mutate_png_encode.py --dry-run   # apply every edit and compile it, no tests

Every edit changes a value or a condition, never an index or a bound of a loop over memory.
Mutants 1-10 are the one-mistake variants of tests/png_oracle.py (VARIANTS)."""
import sys

import mutants

NEW_TESTS = ["tests/test_gpu_png_encode_edges.py"]
OLD_TESTS = ["tests/test_gpu_png.py"]
DESELECT = []
EQUIVALENT = {6, 7, 11}     # no input tells them from the kernel: DESIGN.md §3.21

F = "png.cu"
_PICK = "if (stored_len + 4 <= opt_lenb && can_store) type = 0;"
# (number, what it models, [(file, old, new, occurrences)])
MUTANTS = [
    (1, "smaller()'s depth tiebreak <= made <", [
        (F, "w.depth[n] <= w.depth[m]);", "w.depth[n] < w.depth[m]);", 1)]),
    # 2, the fix-up without `bl_count[max_length]--`, is not built: the counts then name one
    # more leaf per step than the tree has, and the reassignment reads heap slots below the tree
    # that nothing wrote (png_oracle's overflow_keep_max shows the edge images change)
    (3, "the fix-up's search starts at max_length (bit-length tree; the literal tree's would "
        "write bl_count[16])", [
        (F, "      int bits = max_length - 1;", "      int bits = max_length - (kind != 2);", 1)]),
    (4, "a dummy node is always 0", [
        (F, "const int node = max_code < 2 ? ++max_code : 0;", "const int node = 0;", 1)]),
    (5, "the stored pick stored_len + 4 <= opt_lenb made <", [
        (F, _PICK, _PICK.replace("<=", "<"), 1)]),
    (6, "static_lenb <= opt_lenb made < (equivalent: a tie leaves opt_lenb equal either way)", [
        (F, "if (static_lenb <= opt_lenb) opt_lenb", "if (static_lenb < opt_lenb) opt_lenb", 1)]),
    (7, "the static pick == made <= (equivalent: opt_lenb <= static_lenb there)", [
        (F, "else if (static_lenb == opt_lenb) type = 1;",
         "else if (static_lenb <= opt_lenb) type = 1;", 1)]),
    (8, "a byte tie of static and dynamic coding picks dynamic", [
        (F, "else if (static_lenb == opt_lenb) type = 1;",
         "else if (static_lenb < (opt_len + 3 + 7) >> 3) type = 1;", 1)]),
    (9, "walk_tree's min_count of 4 made 3", [
        (F, "max_count = 7, min_count = 4;", "max_count = 7, min_count = 3;", 2)]),
    (10, "a stretch's remainder matched only when r > 3", [
        (F, "else if (r >= 3) code = k == full", "else if (r > 3) code = k == full", 1)]),
    (11, "the window's refusal ignored (equivalent: it never refuses a cheapest stored block)", [
        (F, _PICK, _PICK.replace("&& can_store", "&& true"), 1)]),
    (12, "the Adler-32 weight n - i reduced mod 65520", [
        (F, "(unsigned(T.n - i)) % kMod", "(unsigned(T.n - i)) % (kMod - 1)", 1)]),
    (13, "the Adler-32 trailer written least significant byte first", [
        (F, "v = (unsigned char)(adler >> (24 - 8 * (zi - 2 - dlen)));",
         "v = (unsigned char)(adler >> (8 * (zi - 2 - dlen)));", 1)]),
    (14, "the IDAT length field kept to 13 bits (a full chunk's 8192 reads 0)", [
        (F, "dst[i] = (unsigned char)(len >> (24 - 8 * i));",
         "dst[i] = (unsigned char)((len & 0x1FFF) >> (24 - 8 * i));", 1)]),
]


if __name__ == "__main__":
    mutants.main(sys.modules[__name__])
