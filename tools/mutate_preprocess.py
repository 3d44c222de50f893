#!/usr/bin/env python
"""Do the pre-processing tests notice a subtly wrong kernel?  Fourteen mutants of csrc/mold.cu and
csrc/anchors.cu, each one textual edit that computes wrong VALUES only (no mutant indexes out
of bounds), each built as its own library and put under the tests:

    python tools/mutate_preprocess.py             # on a machine with the GPU
    python tools/mutate_preprocess.py --dry-run   # apply every edit and compile it, no tests

For each mutant: csrc/ is copied to a temporary directory and edited there (a pattern that is
not found exactly as often as stated is an error), the copy is built next to the real library
through build.py's MRX_LIB_NAME hook, and the new test files (test_gpu_cv2_resize, test_gpu_mold,
test_gpu_anchors) and the old one (test_gpu_anchors_mold) each run once in a subprocess with
MRX_LIB naming the mutant.  One table row per mutant: did the new tests fail, did the old ones.
The temporary directory and the mutant library are removed at the end; the repository's own
build is not touched.  A development script: no test imports it."""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from matterport_maskrcnn_with_tensorflow_serving_b200 import build as B  # noqa: E402

NEW_TESTS = {"mold.cu/resize": "tests/test_gpu_cv2_resize.py",
             "mold.cu/mold": "tests/test_gpu_mold.py",
             "anchors.cu": "tests/test_gpu_anchors.py"}
OLD_TESTS = "tests/test_gpu_anchors_mold.py"
# the 2.19 GB sources need 4.3 GB of device memory and no mutant needs them
DESELECT = ["--deselect", "tests/test_gpu_cv2_resize.py::test_source_past_2g_bytes"]

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

# (number, what it models, target, [(old, new, occurrences)])
MUTANTS = [
    (1, "mold: one multiply-add contracted into an FMA", "mold.cu/mold", [
        ("t = __dadd_rn(t, __dmul_rn(__dmul_rn(c11, zy.w1), zx.w1));",
         "t = fma(__dmul_rn(c11, zy.w1), zx.w1, t);", 1)]),
    (2, "mold: the four products summed pairwise", "mold.cu/mold", [
        (ZOOM_SUM, ZOOM_SUM_PAIRWISE, 1)]),
    (3, "mold: the source coordinate from one FMA", "mold.cu/mold", [
        ("__dsub_rn(__dmul_rn(static_cast<double>(k) + 0.5, zoom), 0.5);",
         "fma(static_cast<double>(k) + 0.5, zoom, -0.5);", 1)]),
    (4, "mold: uint8 by rounding instead of truncation", "mold.cu/mold", [
        ("static_cast<unsigned char>(static_cast<int>(t));",
         "static_cast<unsigned char>(__double2int_rn(t));", 1)]),
    (5, "mold: float32 output as float(px) - float(mean)", "mold.cu/mold", [
        ("out[i * 3 + c] = static_cast<TOut>(v);",
         "out[i * 3 + c] = sizeof(TOut) == 4 ? static_cast<TOut>(__fsub_rn("
         "static_cast<float>(px[c]), static_cast<float>(mean[c]))) : static_cast<TOut>(v);", 1)]),
    # the loop bound is kept: later trips visit other pixels, none outside the image
    (6, "mold and resize: grid stride off by one", "mold.cu/resize", [
        ("i += static_cast<long long>(gridDim.x) * kMoldThreads)",
         "i += static_cast<long long>(gridDim.x) * kMoldThreads + 1)", 2)]),
    (7, "resize: area shortcut when either axis is 2x", "mold.cu/resize", [
        ("fabs(scale_x - 2.0) < eps && fabs(scale_y - 2.0) < eps;",
         "fabs(scale_x - 2.0) < eps || fabs(scale_y - 2.0) < eps;", 1),
        (AREA_LOADS, AREA_LOADS_CLAMPED, 1),
        ("(p0[c] + p0[3 + c] + p1[c] + p1[3 + c] + 2) >> 2",
         "(p0[c] + p0[ax + c] + p1[c] + p1[ax + c] + 2) >> 2", 1)]),
    (8, "resize: coefficients truncated, not cvRound", "mold.cu/resize", [
        ("= __float2int_rn(__fmul_rn(", "= __float2int_rz(__fmul_rn(", 2)]),
    (9, "resize: coordinate kept in double", "mold.cu/resize", [
        ("  float f = __double2float_rn(__dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), "
         "0.5));\n  int s = __float2int_rd(f);\n  f = __fsub_rn(f, static_cast<float>(s));\n",
         "  const double fd = __dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), 0.5);\n"
         "  int s = __double2int_rd(fd);\n"
         "  float f = __double2float_rn(__dsub_rn(fd, static_cast<double>(s)));\n", 1)]),
    (10, "resize: y weights clamped like x weights", "mold.cu/resize", [
        ("cv_lin_coef(dy, scale_y, sh, false);", "cv_lin_coef(dy, scale_y, sh, true);", 1)]),
    (11, "resize: vertical pass rounds with + 1", "mold.cu/resize", [
        ("((cy.a1 * (S1 >> 4)) >> 16) + 2) >> 2;", "((cy.a1 * (S1 >> 4)) >> 16) + 1) >> 2;", 1)]),
    # every image read with the sizes of image 0: run only on batches whose image 0 is the
    # smallest, so that every read stays inside its own slot
    (12, "resize batch: sizes of image 0 for every image", "batch", [
        ("sh = src_hw[2 * b];", "sh = src_hw[0];", 1),
        ("sw = src_hw[2 * b + 1];", "sw = src_hw[1];", 1)]),
    # (halving as a multiply is exact, so 0.5 * h as an FMA operand would be an equivalent mutant)
    # The reciprocal moves the float64 quotient by at most one ulp, which changes the float32
    # only for a quotient on a float32 rounding tie: about one value in 2^29, so no sweep meets
    # one; test_gpu_anchors.py::test_division_not_reciprocal constructs such scales.
    (13, "anchors: multiply by the reciprocal instead of dividing", "anchors.cu", [
        ("__ddiv_rn(y1, hm1)", "__dmul_rn(y1, __ddiv_rn(1.0, hm1))", 1),
        ("__ddiv_rn(x1, wm1)", "__dmul_rn(x1, __ddiv_rn(1.0, wm1))", 1),
        ("__ddiv_rn(__dsub_rn(y2, 1.0), hm1)",
         "__dmul_rn(__dsub_rn(y2, 1.0), __ddiv_rn(1.0, hm1))", 1),
        ("__ddiv_rn(__dsub_rn(x2, 1.0), wm1)",
         "__dmul_rn(__dsub_rn(x2, 1.0), __ddiv_rn(1.0, wm1))", 1)]),
    (14, "anchors: ratio and x swapped in the row decode", "anchors.cu", [
        (ANCHOR_DECODE, ANCHOR_DECODE_SWAPPED, 1)]),
]

BATCH_NEW = ["tests/test_gpu_cv2_resize.py::test_batch_equals_single",
             "tests/test_gpu_mold.py::test_preprocess_input_batch"]


def selections(target):
    """(new, old) pytest selections of a mutant; the file that tests the mutated kernel first,
    since each run stops at its first failure.  None: nothing qualifies."""
    if target == "batch":
        # the old file's batches do not start with their smallest image
        return BATCH_NEW, None
    first = NEW_TESTS[target]
    return [first] + [f for f in NEW_TESTS.values() if f != first], [OLD_TESTS]


def mutate(tmp, edits):
    """A copy of the sources under `tmp`, laid out as in the repository (common.cuh includes
    ../../include/mrx.h), with `edits` applied.  Returns its csrc directory."""
    csrc = os.path.join(tmp, "pkg", "csrc")
    shutil.copytree(B.CSRC, csrc)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
    texts = {}
    for name in ("mold.cu", "anchors.cu"):
        with open(os.path.join(csrc, name)) as f:
            texts[name] = f.read()
    for old, new, count in edits:
        found = sum(text.count(old) for text in texts.values())
        if found != count:
            raise SystemExit(f"pattern found {found} times, not {count}: {old!r}")
        texts = {name: text.replace(old, new) for name, text in texts.items()}
    for name, text in texts.items():
        with open(os.path.join(csrc, name), "w") as f:
            f.write(text)
    return csrc


def build_mutant(number, csrc):
    """lib/libmrx_mutant<number>.so from the sources in `csrc`.  The objects of the unedited
    sources are the real build's (their stamps are digests of file contents, equal here), so
    only the edited file compiles."""
    name = f"libmrx_mutant{number}.so"
    os.environ["MRX_LIB_NAME"] = name
    real_obj = os.path.join(B.LIB_DIR, "obj_libmrx")
    obj_dir = os.path.join(B.LIB_DIR, "obj_" + name[:-3])
    if os.path.isdir(real_obj):
        shutil.copytree(real_obj, obj_dir, dirs_exist_ok=True)
    saved = B.CSRC, B.HEADERS
    # each header where the copy keeps it: csrc/ headers in `csrc`, the others in ../../include
    include = os.path.join(os.path.dirname(os.path.dirname(csrc)), "include")
    B.HEADERS = [os.path.join(csrc if os.path.dirname(h) == B.CSRC else include,
                              os.path.basename(h)) for h in B.HEADERS]
    B.CSRC = csrc
    missing = [h for h in B.HEADERS if not os.path.exists(h)]
    if missing:
        raise SystemExit(f"the copied sources lack {missing}")
    try:
        return B.build()
    finally:
        B.CSRC, B.HEADERS = saved
        del os.environ["MRX_LIB_NAME"]


def remove_mutant(number):
    name = f"libmrx_mutant{number}"
    for path in (os.path.join(B.LIB_DIR, name + ".so"), os.path.join(B.LIB_DIR, name + ".stamp")):
        if os.path.exists(path):
            os.remove(path)
    shutil.rmtree(os.path.join(B.LIB_DIR, "obj_" + name), ignore_errors=True)


def killed(number, selection, log_dir):
    """'survived' when the tests pass against the mutant, 'killed by <test>' when one fails
    on an assertion; a run that ends any other way (a fixture or collection error, a usage
    error) is no verdict and ends the script."""
    if selection is None:
        return "not run"
    # COLUMNS: pytest cuts the summary lines read below to the terminal's width
    env = dict(os.environ, MRX_LIB=f"libmrx_mutant{number}.so", COLUMNS="400")
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-rfE", "-p", "no:cacheprovider",
           *selection, *DESELECT]
    res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    if log_dir:
        tag = "new" if selection[0] != OLD_TESTS else "old"
        with open(os.path.join(log_dir, f"mutant{number}_{tag}.log"), "w") as f:
            f.write(res.stdout[-20000:] + res.stderr[-5000:])
    if res.returncode == 0:
        return "survived"
    summary = [ln for ln in res.stdout.splitlines() if ln.startswith(("FAILED ", "ERROR "))]
    if res.returncode != 1 or len(summary) != 1 or not summary[0].startswith("FAILED ") \
            or " - assert" not in summary[0].lower():
        raise SystemExit(f"mutant {number}: pytest ended with {res.returncode} and no single "
                         f"failed assertion\n{res.stdout[-3000:]}{res.stderr[-3000:]}")
    return "killed by " + summary[0].split(" - ")[0][len("FAILED tests/"):]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--dry-run", action="store_true", help="edit and compile only")
    ap.add_argument("--only", type=int, nargs="*", help="mutant numbers (default: all)")
    ap.add_argument("--logs", help="directory for each run's pytest output")
    args = ap.parse_args()
    if args.logs:
        os.makedirs(args.logs, exist_ok=True)
    B.build()     # the real library, whose objects the mutants share
    rows = []
    for number, what, target, edits in MUTANTS:
        if args.only and number not in args.only:
            continue
        tmp = tempfile.mkdtemp(prefix="mrx_mutant_")
        try:
            path = build_mutant(number, mutate(tmp, edits))
            if args.dry_run:
                rows.append((number, what, "built", "built"))
                assert os.path.exists(path)
            else:
                new, old = selections(target)
                rows.append((number, what, killed(number, new, args.logs),
                             killed(number, old, args.logs)))
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
            remove_mutant(number)
        print("| {} | {} | {} | {} |".format(*rows[-1]), flush=True)
    print("\n| # | mutant | new tests | old tests |\n|---|---|---|---|")
    for row in rows:
        print("| {} | {} | {} | {} |".format(*row))
    survivors = [r[0] for r in rows if r[2] == "survived"]
    if survivors:
        raise SystemExit(f"the new tests let mutants {survivors} live")


if __name__ == "__main__":
    main()
