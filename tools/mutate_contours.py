#!/usr/bin/env python
"""Do the contour tests notice a tracer that is subtly wrong?  Value-only mutants of the kernels
(csrc/contours.cu) and of the NumPy entry's regions (visualize._trace_masks), run by
tools/mutants.py under the new edge tests and the older ones:

    python tools/mutate_contours.py             # on a machine with the GPU
    python tools/mutate_contours.py --dry-run   # apply every edit and compile it, no tests

Every mutant stays in bounds, for one of three reasons:
  * it changes the traced 0/1 image but keeps its zero ring, with cells and pixels changed
    together (1, 2, 8: the region clamp in inst_of, which both passes read).  The clamped region
    still lies inside the image, so no plane byte past the instance's plane is read, the rows stay
    below row_pitch, and the image traced is a padded 0/1 image whose segments form closed cycles
    of at least 4: the count pass sizes every buffer for exactly what the link pass writes;
  * it changes vertex values only (3, 5, 6): the stores go where they went;
  * it changes the contour order key consistently (4): heads, lengths, scan and write all move to
    the cycle's largest segment, still one per cycle, so the contour and vertex counts are those
    of the correct code.
No mutant touches a successor number, a jump record, a scan base or a write offset: a wrong
successor can close cycles shorter than 4 and write past the S/4 contour bound.  Host mutant 7
changes which regions are traced, which the count pass sizes.  None is argued equivalent."""
import sys

import mutants

NEW_TESTS = ["tests/test_gpu_contour_edges.py"]
OLD_TESTS = ["tests/test_gpu_contours.py", "tests/test_gpu_annotate.py"]
DESELECT = []
EQUIVALENT = set()

C = "contours.cu"
CLAMP = "in.g = {max(r.x, 0), max(r.y, 0), min(r.z, H), min(r.w, W)};"
# (number, what it models, [(file, old, new, occurrences)]); file visualize.py: host
MUTANTS = [
    (1, "region x1 ignored: traced from column 0", [
        (C, CLAMP, "in.g = {max(r.x, 0), 0, min(r.z, H), min(r.w, W)};", 1)]),
    (2, "region y2 ignored: traced down to the image's last row", [
        (C, CLAMP, "in.g = {max(r.x, 0), max(r.y, 0), H, min(r.w, W)};", 1)]),
    (3, "vertex rounded through float32", [
        (C, "make_double2(0.5 * h.x, 0.5 * h.y)",
         "make_double2(static_cast<float>(0.5 * h.x), static_cast<float>(0.5 * h.y))", 1)]),
    (4, "contours ordered by their largest segment", [
        (C, "    if (r.y == s) {", "    if (r.z == s) {", 1),
        (C, "    const int m = r.y;", "    const int m = r.z;", 1)]),
    (5, "kLeft vertex into the previous word one pixel left", [
        (C, "v = make_int2(half_units(c - 1, c - 1), half_units(r - 1, r));",
         "v = make_int2(half_units(c - 1, c - 1) - 2 * (jl == 0), half_units(r - 1, r));", 1)]),
    (6, "kBottom vertex one pixel low", [
        (C, "v = make_int2(half_units(c - 1, c), half_units(r, r));",
         "v = make_int2(half_units(c - 1, c), half_units(r + 1, r + 1));", 1)]),
    (7, "host: all-zero boxes traced over the whole image", [
        ("visualize.py", "regions[boxes.reshape(n, -1).any(axis=1)] = (0, 0, H, W)",
         "regions[:] = (0, 0, H, W)", 1)]),
    (8, "instances past counts[b] traced", [
        (C, "const bool empty = k >= p.counts[b] || ", "const bool empty = ", 1)]),
]


if __name__ == "__main__":
    mutants.main(sys.modules[__name__])
