#!/usr/bin/env python
"""Do the mask-expand tests notice a kernel that is off by an ulp?  Ten mutants of the expand
kernels (csrc/expand.cuh, expand_team.cu, unmold.cu, expand_bits.cu, rle.cu), each a textual
edit that changes VALUES only (no mutant indexes out of bounds; none touches the NaN threshold
of the columns outside a box), each built as its own library and put under the tests:

    python tools/mutate_expand.py             # on a machine with the GPU
    python tools/mutate_expand.py --dry-run   # apply every edit and compile it, no tests

For each mutant: csrc/ is copied to a temporary directory and edited there (a pattern that is
not found exactly as often as stated is an error), the copy is built next to the real library
through build.py's MRX_LIB_NAME hook, and the new test file (test_gpu_expand_exact) and the old
ones (test_gpu_unmold, test_gpu_tile_shapes, test_gpu_kernel_paths, test_gpu_pack, test_gpu_rle,
without their multi-GB cases) each run once in a subprocess with MRX_LIB naming the mutant.  One
table row per mutant: did the new tests fail, did the old ones.  The temporary directory and the
mutant library are removed at the end; the repository's own build is not touched.  A development
script: no test imports it."""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from matterport_maskrcnn_with_tensorflow_serving_b200 import build as B  # noqa: E402

NEW_TESTS = ["tests/test_gpu_expand_exact.py"]
OLD_TESTS = ["tests/test_gpu_unmold.py", "tests/test_gpu_tile_shapes.py",
             "tests/test_gpu_kernel_paths.py", "tests/test_gpu_pack.py", "tests/test_gpu_rle.py"]
# the cases that need gigabytes of device memory (and minutes); no mutant needs them
DESELECT = [a for t in ("tests/test_gpu_unmold.py::test_full_size_properties",
                        "tests/test_gpu_unmold.py::test_config4_4k_shape_properties",
                        "tests/test_gpu_unmold.py::test_exhaustive_config4_4k",
                        "tests/test_gpu_rle.py::test_rle_full_size_batch")
            for a in ("--deselect", t)]
FILES = ("expand.cuh", "expand_team.cu", "unmold.cu", "expand_bits.cu", "rle.cu")

SRC_FLOOR = """\
  int rem = A - i * D;
  if (rem < 0) {
    --i;
    rem += D;
  } else if (rem >= D) {
    ++i;
    rem -= D;
  }
  return {i, rem};
"""
SRC_FLOOR_UNCORRECTED = """\
  int rem = A - i * D;
  return {i, rem};
"""

# (number, what it models, [(file, old, new, occurrences)])
MUTANTS = [
    (1, "team kernel: > 0.5 instead of >= 0.5", [
        ("expand_team.cu", "if (v >= thr)", "if (v > thr)", 1),
        ("expand_team.cu", "if (v >= 0.5f && colvalid)", "if (v > 0.5f && colvalid)", 1)]),
    (2, "generic kernel: > 0.5 instead of >= 0.5", [
        ("unmold.cu", "if (lerp(e.wy, ht, hb) >= 0.5f && off < ulen)",
         "if (lerp(e.wy, ht, hb) > 0.5f && off < ulen)", 1)]),
    (3, "packed kernel: > 0.5 instead of >= 0.5", [
        ("expand_bits.cu", "__ballot_sync(0xffffffffu, v >= thr[c])",
         "__ballot_sync(0xffffffffu, v > thr[c])", 1)]),
    (4, "RLE kernel: > 0.5 instead of >= 0.5", [
        ("rle.cu", "cur = v >= thr;", "cur = v > thr;", 1),
        ("rle.cu", "vl >= 0.5f;", "vl > 0.5f;", 1)]),
    (5, "every kernel: lerp as a multiply and an add", [
        ("expand.cuh", "return fmaf(w, hi - lo, lo);", "return __fadd_rn(__fmul_rn(w, hi - lo), lo);",
         1)]),
    (6, "team kernel: 1/D of the columns rounded toward zero", [
        ("expand_team.cu", "e.invD = __fdiv_rn(1.0f, static_cast<float>(2 * (bx.w - bx.y)));",
         "e.invD = __frcp_rz(static_cast<float>(2 * (bx.w - bx.y)));", 1)]),
    (7, "generic kernel: 1/D of the columns rounded toward zero", [
        ("unmold.cu", "e.invD = __fdiv_rn(1.0f, static_cast<float>(e.D));",
         "e.invD = __frcp_rz(static_cast<float>(e.D));", 1)]),
    (8, "packed kernel: 1/D of the columns rounded toward zero", [
        ("expand_bits.cu", "const float invD = __fdiv_rn(1.0f, static_cast<float>(D));",
         "const float invD = __frcp_rz(static_cast<float>(D));", 1)]),
    (9, "RLE kernel: 1/D of the columns rounded toward zero", [
        ("rle.cu", "const float invD = __fdiv_rn(1.0f, static_cast<float>(D));",
         "const float invD = __frcp_rz(static_cast<float>(D));", 1)]),
    # the estimate is never too high (test_expand_oracle.py): without the correction a too-low
    # floor keeps rem = D, weight ~1 on the row / column below, every index still in range
    (10, "every kernel: src_floor without its correction", [
        ("expand.cuh", SRC_FLOOR, SRC_FLOOR_UNCORRECTED, 1)]),
]


def mutate(tmp, edits):
    """A copy of the sources under `tmp`, laid out as in the repository (common.cuh includes
    ../../include/mrx.h), with `edits` applied.  Returns its csrc directory."""
    csrc = os.path.join(tmp, "pkg", "csrc")
    shutil.copytree(B.CSRC, csrc)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
    texts = {}
    for name in FILES:
        with open(os.path.join(csrc, name)) as f:
            texts[name] = f.read()
    for name, old, new, count in edits:
        found = texts[name].count(old)
        if found != count:
            raise SystemExit(f"{name}: pattern found {found} times, not {count}: {old!r}")
        texts[name] = texts[name].replace(old, new)
    for name, text in texts.items():
        with open(os.path.join(csrc, name), "w") as f:
            f.write(text)
    return csrc


def build_mutant(number, csrc):
    """lib/libmrx_mutant<number>.so from the sources in `csrc`.  The objects of the unedited
    sources are the real build's (their stamps are digests of file contents and headers, equal
    here), so only what the edit reaches compiles."""
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


def killed(number, selection, tag, log_dir):
    """'survived' when the tests pass against the mutant, 'killed by <test>' when one fails
    on an assertion; a run that ends any other way (a fixture or collection error, a usage
    error) is no verdict and ends the script."""
    # COLUMNS: pytest cuts the summary lines read below to the terminal's width
    env = dict(os.environ, MRX_LIB=f"libmrx_mutant{number}.so", COLUMNS="400")
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-rfE", "-p", "no:cacheprovider",
           *selection, *DESELECT]
    res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    if log_dir:
        with open(os.path.join(log_dir, f"mutant{number}_{tag}.log"), "w") as f:
            f.write(res.stdout[-20000:] + res.stderr[-5000:])
    if res.returncode == 0:
        return "survived"
    summary = [ln for ln in res.stdout.splitlines() if ln.startswith(("FAILED ", "ERROR "))]
    if res.returncode != 1 or len(summary) != 1 or not summary[0].startswith("FAILED ") \
            or " - assert" not in summary[0].lower() and " - failed" not in summary[0].lower():
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
    for number, what, edits in MUTANTS:
        if args.only and number not in args.only:
            continue
        tmp = tempfile.mkdtemp(prefix="mrx_mutant_")
        try:
            path = build_mutant(number, mutate(tmp, edits))
            if args.dry_run:
                rows.append((number, what, "built", "built"))
                assert os.path.exists(path)
            else:
                rows.append((number, what, killed(number, NEW_TESTS, "new", args.logs),
                             killed(number, OLD_TESTS, "old", args.logs)))
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
