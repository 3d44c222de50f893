#!/usr/bin/env python
"""Do the polygon tests notice a rasteriser that is subtly wrong?  Value-only mutants of the
kernels (csrc/polygons.cu) and of the host packing (engine.pack_polygons), run by
tools/mutants.py under the new edge tests and the older ones:

    python tools/mutate_polygons.py             # on a machine with the GPU
    python tools/mutate_polygons.py --dry-run   # apply every edit and compile it, no tests

No mutant indexes out of bounds or shifts by 32 or more: bucket stores stay clamped to the host's
bound whatever it is.  Mutants marked equivalent are argued so in DESIGN §3.16 (the junction pair
never toggles a column inside the image; no column holds an odd number of toggles); they are
still run, and their row says whether the tests agree."""
import sys

import mutants

NEW_TESTS = ["tests/test_gpu_polygon_edges.py"]
OLD_TESTS = ["tests/test_gpu_polygons.py", "tests/test_gpu_cocoeval_boundary.py"]
DESELECT = []
EQUIVALENT = {10, 14, 18}

P = "polygons.cu"
# (number, what it models, [(file, old, new, occurrences)]); file engine.py: host
MUTANTS = [
    (1, "minor_at: a + s*t + .5 with a + s*t contracted into an FMA", [
        (P, "__dadd_rn(__dadd_rn(static_cast<double>(a),\n"
            "                                            __dmul_rn(s, static_cast<double>(t))), 0.5)",
         "__dadd_rn(__fma_rn(s, static_cast<double>(t), static_cast<double>(a)), 0.5)", 1)]),
    (2, "Edge: s = diff * (1/n) in place of __ddiv_rn", [
        (P, "__ddiv_rn(static_cast<double>(xmaj ? ye - ys : xe - xs),\n"
            "                                 static_cast<double>(n))",
         "__dmul_rn(static_cast<double>(xmaj ? ye - ys : xe - xs),\n"
         "                                 __drcp_rn(static_cast<double>(n)))", 1)]),
    (3, "toggle_row: (vmin + 3) / 5", [(P, "(vmin + 2) / 5", "(vmin + 3) / 5", 1)]),
    (4, "toggle_row: clamped at H - 1", [
        (P, "min(static_cast<long long>(H), (vmin", "min(static_cast<long long>(H - 1), (vmin", 1)]),
    (5, "x-major pair: the row from the first point (u = c) only", [
        (P, "emit(toggle_row(min(e.v(c - e.xs), e.v(c + 1 - e.xs)), H))",
         "emit(toggle_row(e.v(c - e.xs), H))", 1)]),
    (6, "y-major pair: the row e.ys + hi", [
        (P, "emit(toggle_row(e.ys + lo, H))", "emit(toggle_row(e.ys + hi, H))", 1)]),
    (7, "y-major pair: the `want` test inverted", [
        (P, "rising != e.flip ? c + 1 : c", "rising == e.flip ? c + 1 : c", 1)]),
    (8, "y-major pair: the point e.flip ? hi : lo", [
        (P, "e.u(e.flip ? lo : hi) == want", "e.u(e.flip ? hi : lo) == want", 1)]),
    (9, "edge cull one unit past the tightest correct one (c = min x, c + 1 = max x culled)", [
        (P, "min(a.x, b.x)) - 3", "min(a.x, b.x)) + 2", 1),
        (P, "max(a.x, b.x)) + 3", "max(a.x, b.x)) - 2", 1)]),
    (10, "column carry from the pass-local prefix", [
        (P, "cy[X] = static_cast<unsigned char>(ex & 1);",
         "cy[X] = static_cast<unsigned char>((ex - done) & 1);", 1)]),
    (11, "bucket positions without the earlier passes' toggles", [
        (P, "long long q = t0 + ex;", "long long q = t0 + ex - done;", 1)]),
    (12, "parts XORed in place of ORed", [(P, "word |= w;", "word ^= w;", 1)]),
    (13, "band: a toggle applied one row late", [
        (P, "w ^= 0xFFFFFFFFu << (y - y0);", "w ^= (0xFFFFFFFFu << (y - y0)) << 1;", 1)]),
    (14, "the junction pair's toggle never emitted", [
        (P, "if (fu != pu && (fu < pu", "if (false && fu != pu && (fu < pu", 1)]),
    (15, "host: vertices scaled with np.floor for np.trunc", [
        ("engine.py", "sc = np.trunc(np.add(np.multiply(5.0, xy), 0.5))",
         "sc = np.floor(np.add(np.multiply(5.0, xy), 0.5))", 1)]),
    (16, "host: box corners as scaled x plus scaled w", [
        ("engine.py", "            xe, ye = x + w, y + h\n",
         "            xe = (np.trunc(5.0 * x + .5) + np.trunc(5.0 * w + .5)) / 5.0\n"
         "            ye = (np.trunc(5.0 * y + .5) + np.trunc(5.0 * h + .5)) / 5.0\n", 1)]),
    (17, "host: toggle bound min(W, (|dx| + 3) // 5) per edge", [
        ("engine.py", "np.minimum(W[vpart], (d[:, 0] + 2) // 5 + 1) + 1",
         "np.minimum(W[vpart], (d[:, 0] + 3) // 5)", 1)]),
    (18, "host: toggle bound without the junction's + 1", [
        ("engine.py", "np.minimum(W[vpart], (d[:, 0] + 2) // 5 + 1) + 1",
         "np.minimum(W[vpart], (d[:, 0] + 2) // 5 + 1)", 1)]),
]


if __name__ == "__main__":
    mutants.main(sys.modules[__name__])
