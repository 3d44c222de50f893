#!/usr/bin/env python
"""Do the scoring tests notice a kernel that breaks a tie or a bound the other way?  Fifteen
mutants of the scoring kernels (csrc/cocoeval.cu, overlaps.cu, planes.cuh), each a textual edit
that changes VALUES only (no mutant indexes out of bounds), each built as its own library and put
under the tests:

    python tools/mutate_eval.py             # on a machine with the GPU
    python tools/mutate_eval.py --dry-run   # apply every edit and compile it, no tests

For each mutant: csrc/ is copied to a temporary directory and edited there (a pattern that is
not found exactly as often as stated is an error), the copy is built next to the real library
through build.py's MRX_LIB_NAME hook, and the new test file (test_gpu_score_edges) and the old
ones (test_gpu_cocoeval, test_gpu_cocoeval_bbox, test_gpu_cocoeval_boundary, test_gpu_eval,
test_gpu_lvis) each run once in a subprocess with MRX_LIB naming the mutant.  One table row per
mutant: did the new tests fail, did the old ones.  The temporary directory and the mutant library
are removed at the end; the repository's own build is not touched.  A development script: no
test imports it."""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from matterport_maskrcnn_with_tensorflow_serving_b200 import build as B  # noqa: E402

NEW_TESTS = ["tests/test_gpu_score_edges.py"]
OLD_TESTS = ["tests/test_gpu_cocoeval.py", "tests/test_gpu_cocoeval_bbox.py",
             "tests/test_gpu_cocoeval_boundary.py", "tests/test_gpu_eval.py",
             "tests/test_gpu_lvis.py"]
DESELECT = []
FILES = ("cocoeval.cu", "overlaps.cu", "planes.cuh")

# (number, what it models, [(file, old, new, occurrences)])
MUTANTS = [
    (1, "coco_match: lane ties to the smaller j (key > best)", [
        ("cocoeval.cu", "if (key >= best || bj < 0)", "if (key > best || bj < 0)", 1)]),
    (2, "coco_match: ties across lanes to the smaller j (oj < bj)", [
        ("cocoeval.cu", "(ok == best && oj > bj)", "(ok == best && oj < bj)", 1)]),
    (3, "coco_match: strict IoU threshold (v > thr)", [
        ("cocoeval.cu", "if (!(v >= thr)) continue;", "if (!(v > thr)) continue;", 1)]),
    (4, "coco_match: ground truth at the lower area bound ignored (ga <= lo)", [
        ("cocoeval.cu", "crowd || ga < lo || ga > hi", "crowd || ga <= lo || ga > hi", 1)]),
    (5, "coco_match: unmatched detection at the upper bound ignored (da >= hi)", [
        ("cocoeval.cu", "ig = da < lo || da > hi;", "ig = da < lo || da >= hi;", 1)]),
    (6, "coco_match: crowd instances matched only once", [
        ("cocoeval.cu", "if (!crowd && (s_matched[j >> 5] >> (j & 31) & 1u)) continue;",
         "if ((s_matched[j >> 5] >> (j & 31) & 1u)) continue;", 1)]),
    (7, "mask_match: NaN keyed as IoU 0, below every number", [
        ("overlaps.cu", "key = (2ull << 62) | static_cast<unsigned>(j);",
         "key = (1ull << 62) | static_cast<unsigned>(j);", 1)]),
    (8, "mask_match: strict IoU threshold (> thr)", [
        ("overlaps.cu", "static_cast<double>(v) >= thr &&", "static_cast<double>(v) > thr &&", 1)]),
    (9, "mask_match: IoU ties to the smaller j", [
        ("overlaps.cu", "static_cast<unsigned>(j);", "(0xFFFFu - static_cast<unsigned>(j));", 2),
        ("overlaps.cu", "static_cast<int>(best & 0xFFFFu)",
         "static_cast<int>(0xFFFFu - (best & 0xFFFFu))", 1)]),
    (10, "mask_rank: score ties to the smaller index (k < i)", [
        ("overlaps.cu", "(tie && k > i)", "(tie && k < i)", 1)]),
    (11, "rle_iou: crowd union from the ground truth's area (a2)", [
        ("cocoeval.cu", "const long long u = crowd ? a1 : a1 + a2 - inter;",
         "const long long u = crowd ? a2 : a1 + a2 - inter;", 1)]),
    (12, "and_count: first-byte mask from (x1 + 1) & 7", [
        ("planes.cuh", "first = 0xFFu >> (x1 & 7)", "first = 0xFFu >> ((x1 + 1) & 7)", 1)]),
    (13, "and_count: last-byte mask shifted by one", [
        ("planes.cuh", "last = (0xFFu << (7 - ((x2 - 1) & 7))) & 0xFFu",
         "last = (0xFFu << (8 - ((x2 - 1) & 7))) & 0xFFu", 1)]),
    (14, "coco_box_iou: da + g[2]*g[3] contracted into an fma", [
        ("cocoeval.cu", "__dsub_rn(__dadd_rn(da, __dmul_rn(g[2], g[3])), inter)",
         "__dsub_rn(__fma_rn(g[2], g[3], da), inter)", 1)]),
    (15, "LVIS keep: the cut by rank in the category instead of the walk", [
        ("cocoeval.cu", "int b, int ci, int,", "int b, int ci, int rank,", 1),
        ("cocoeval.cu", "walk < p.max_det &&", "rank < p.max_det &&", 1)]),
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
    ap.add_argument("--new-only", action="store_true",
                    help="run only the new tests (the old ones take minutes per survivor)")
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
                             "not run" if args.new_only else
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
