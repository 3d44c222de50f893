#!/usr/bin/env python
"""Do the annotation tests notice boxes, outlines or captions that are subtly wrong?  Value-only
mutants of the kernels (csrc/annotate.cu) and of the host captions and colours (visualize.py),
run by tools/mutants.py under the new tests and the overlay's older ones:

    python tools/mutate_annotate.py             # on a machine with the GPU
    python tools/mutate_annotate.py --dry-run   # apply every edit and compile it, no tests

No mutant writes outside a key plane or an image: clipping mutants clamp onto the border instead
of dropping the pixel.  None is argued equivalent."""
import sys

import mutants

NEW_TESTS = ["tests/test_host_annotate.py", "tests/test_gpu_annotate.py"]
OLD_TESTS = ["tests/test_gpu_composite.py", "tests/test_gpu_contours.py"]
# the table test imports tools/, which the host mutants' copy of the tree does not hold
DESELECT = ["tests/test_host_annotate.py::test_mutant_table_matches_the_sources"]
EQUIVALENT = set()

A = "annotate.cu"
V = "visualize.py"
# (number, what it models, [(file, old, new, occurrences)]); file visualize.py: host
MUTANTS = [
    (1, "colour table: 255 c rounded half up instead of cvRound's half to even", [
        (V, "v = np.rint(255.0 * float(col[c]))", "v = np.floor(255.0 * float(col[c]) + 0.5)", 1)]),
    (2, "box: right edge at x2 - 1", [
        (A, "xb = max(bx.y, bx.w);", "xb = max(bx.y, bx.w - 1);", 1)]),
    (3, "segment rule: end points rounded half down", [
        (A, "return (__double2int_rn(2.0 * u) + 1) >> 1;", "return __double2int_rn(2.0 * u) >> 1;",
         1)]),
    (4, "segment clip ignored: end points outside the image clamped onto its border", [
        (A, "const int x = round_half_up(p.x), y = round_half_up(p.y);\n"
            "    if (x < 0 || x >= W || y < 0 || y >= H) continue;",
         "const int x = min(max(round_half_up(p.x), 0), W - 1),\n"
         "              y = min(max(round_half_up(p.y), 0), H - 1);", 1)]),
    (5, "box clip ignored: a bottom edge at y2 == H clamped onto row H - 1", [
        (A, "if (yb >= 0 && yb < H) atomicMax(kp + static_cast<long long>(yb) * W + x, key);",
         "atomicMax(kp + static_cast<long long>(min(max(yb, 0), H - 1)) * W + x, key);", 1)]),
    (6, "priority by min: the earlier instance wins", [
        (A, "const int key = k + 1;", "const int key = R - k;", 1),
        (A, "static_cast<long long>(y) * W + x, k + 1);", "static_cast<long long>(y) * W + x, R - k);",
         1),
        (A, "tab + (key - 1) * 3", "tab + (R - key) * 3", 1)]),
    (7, "captions under the outlines: the stencils blitted before the keys resolve", [
        (A, "  if (P > 0) {\n    annotate_caption_kernel", "  if (false) {\n    annotate_caption_kernel",
         1),
        (A, "  annotate_resolve_kernel<<<pixel_grid(max_pixels, B, dev), kThreads, 0, st>>>(",
         "  if (P > 0)\n    annotate_caption_kernel<<<P, kThreads, 0, st>>>(d_geom, d_images, "
         "d_image_off, d_stencils, d_patches, B);\n"
         "  annotate_resolve_kernel<<<pixel_grid(max_pixels, B, dev), kThreads, 0, st>>>(", 1)]),
    (8, "caption at y1 + 7", [(V, "CAPTION_DY = 8 ", "CAPTION_DY = 7 ", 1)]),
    (9, "score 0 captioned as 0.000", [
        (V, '"{} {:.3f}".format(label, score) if score else label',
         '"{} {:.3f}".format(label, score) if score is not None else label', 1)]),
    (10, "show_bbox ignored", [(A, "if (show_bbox) {", "if (true) {", 1)]),
]


if __name__ == "__main__":
    mutants.main(sys.modules[__name__])
