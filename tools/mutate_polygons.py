#!/usr/bin/env python
"""Do the polygon tests notice a rasteriser that is subtly wrong?  Value-only mutants of the
kernels (csrc/polygons.cu) and of the host packing (engine.pack_polygons), each put under the new
edge tests and the older ones:

    python tools/mutate_polygons.py             # on a machine with the GPU
    python tools/mutate_polygons.py --dry-run   # apply every edit and compile it, no tests

Kernel mutants are built as their own library through tools/mutate_eval.py's copy-and-build
(build.py's MRX_LIB_NAME hook) and selected with MRX_LIB.  Host mutants run on a temporary copy of
the package and the tests, with the real library and header linked in.  No mutant indexes out of
bounds or shifts by 32 or more: bucket stores stay clamped to the host's bound whatever it is.
Mutants marked equivalent are argued so in DESIGN §3.16 (the junction pair never toggles a column
inside the image; no column holds an odd number of toggles); they are still run, and their row
says whether the tests agree.  The repository's sources and build are not touched.  A
development script: no test imports it."""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mutate_eval as ME  # noqa: E402
from matterport_maskrcnn_with_tensorflow_serving_b200 import build as B  # noqa: E402

NEW_TESTS = ["tests/test_gpu_polygon_edges.py"]
OLD_TESTS = ["tests/test_gpu_polygons.py", "tests/test_gpu_cocoeval_boundary.py"]
PKG = "matterport_maskrcnn_with_tensorflow_serving_b200"

P = "polygons.cu"
# (number, what it models, equivalent, [(file, old, new, occurrences)]); file engine.py: host
MUTANTS = [
    (1, "minor_at: a + s*t + .5 with a + s*t contracted into an FMA", False, [
        (P, "__dadd_rn(__dadd_rn(static_cast<double>(a),\n"
            "                                            __dmul_rn(s, static_cast<double>(t))), 0.5)",
         "__dadd_rn(__fma_rn(s, static_cast<double>(t), static_cast<double>(a)), 0.5)", 1)]),
    (2, "Edge: s = diff * (1/n) in place of __ddiv_rn", False, [
        (P, "__ddiv_rn(static_cast<double>(xmaj ? ye - ys : xe - xs),\n"
            "                                 static_cast<double>(n))",
         "__dmul_rn(static_cast<double>(xmaj ? ye - ys : xe - xs),\n"
         "                                 __drcp_rn(static_cast<double>(n)))", 1)]),
    (3, "toggle_row: (vmin + 3) / 5", False, [(P, "(vmin + 2) / 5", "(vmin + 3) / 5", 1)]),
    (4, "toggle_row: clamped at H - 1", False, [
        (P, "min(static_cast<long long>(H), (vmin", "min(static_cast<long long>(H - 1), (vmin", 1)]),
    (5, "x-major pair: the row from the first point (u = c) only", False, [
        (P, "emit(toggle_row(min(e.v(c - e.xs), e.v(c + 1 - e.xs)), H))",
         "emit(toggle_row(e.v(c - e.xs), H))", 1)]),
    (6, "y-major pair: the row e.ys + hi", False, [
        (P, "emit(toggle_row(e.ys + lo, H))", "emit(toggle_row(e.ys + hi, H))", 1)]),
    (7, "y-major pair: the `want` test inverted", False, [
        (P, "rising != e.flip ? c + 1 : c", "rising == e.flip ? c + 1 : c", 1)]),
    (8, "y-major pair: the point e.flip ? hi : lo", False, [
        (P, "e.u(e.flip ? lo : hi) == want", "e.u(e.flip ? hi : lo) == want", 1)]),
    (9, "edge cull one unit past the tightest correct one (c = min x, c + 1 = max x culled)",
     False, [(P, "min(a.x, b.x)) - 3", "min(a.x, b.x)) + 2", 1),
             (P, "max(a.x, b.x)) + 3", "max(a.x, b.x)) - 2", 1)]),
    (10, "column carry from the pass-local prefix", True, [
        (P, "cy[X] = static_cast<unsigned char>(ex & 1);",
         "cy[X] = static_cast<unsigned char>((ex - done) & 1);", 1)]),
    (11, "bucket positions without the earlier passes' toggles", False, [
        (P, "long long q = t0 + ex;", "long long q = t0 + ex - done;", 1)]),
    (12, "parts XORed in place of ORed", False, [(P, "word |= w;", "word ^= w;", 1)]),
    (13, "band: a toggle applied one row late", False, [
        (P, "w ^= 0xFFFFFFFFu << (y - y0);", "w ^= (0xFFFFFFFFu << (y - y0)) << 1;", 1)]),
    (14, "the junction pair's toggle never emitted", True, [
        (P, "if (fu != pu && (fu < pu", "if (false && fu != pu && (fu < pu", 1)]),
    (15, "host: vertices scaled with np.floor for np.trunc", False, [
        ("engine.py", "sc = np.trunc(np.add(np.multiply(5.0, xy), 0.5))",
         "sc = np.floor(np.add(np.multiply(5.0, xy), 0.5))", 1)]),
    (16, "host: box corners as scaled x plus scaled w", False, [
        ("engine.py", "            xe, ye = x + w, y + h\n",
         "            xe = (np.trunc(5.0 * x + .5) + np.trunc(5.0 * w + .5)) / 5.0\n"
         "            ye = (np.trunc(5.0 * y + .5) + np.trunc(5.0 * h + .5)) / 5.0\n", 1)]),
    (17, "host: toggle bound min(W, (|dx| + 3) // 5) per edge", False, [
        ("engine.py", "np.minimum(W[vpart], (d[:, 0] + 2) // 5 + 1) + 1",
         "np.minimum(W[vpart], (d[:, 0] + 3) // 5)", 1)]),
    (18, "host: toggle bound without the junction's + 1", True, [
        ("engine.py", "np.minimum(W[vpart], (d[:, 0] + 2) // 5 + 1) + 1",
         "np.minimum(W[vpart], (d[:, 0] + 2) // 5 + 1)", 1)]),
]


def apply(path, edits):
    with open(path) as f:
        text = f.read()
    for _, old, new, count in edits:
        found = text.count(old)
        if found != count:
            raise SystemExit(f"{os.path.basename(path)}: pattern found {found} times, not "
                             f"{count}: {old!r}")
        text = text.replace(old, new)
    with open(path, "w") as f:
        f.write(text)


def host_tree(tmp, edits):
    """A root under `tmp` with the package (engine.py edited), tests/, include/ and oracle/ as
    the repository has them, and the package's lib/ linked to the real build."""
    pkg = os.path.join(tmp, PKG)
    shutil.copytree(os.path.join(ROOT, PKG), pkg,
                    ignore=shutil.ignore_patterns("lib", "__pycache__"))
    os.symlink(B.LIB_DIR, os.path.join(pkg, "lib"))
    shutil.copytree(os.path.join(ROOT, "tests"), os.path.join(tmp, "tests"),
                    ignore=shutil.ignore_patterns("__pycache__"))
    for name in ("include", "oracle"):
        os.symlink(os.path.join(ROOT, name), os.path.join(tmp, name))
    apply(os.path.join(pkg, "engine.py"), edits)
    return tmp


def run_tests(selection, cwd, env, tag, number, log_dir):
    """'survived', or 'killed by <test>' when exactly one test fails on an assertion."""
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-rfE", "-p", "no:cacheprovider",
           *selection]
    res = subprocess.run(cmd, cwd=cwd, env=dict(os.environ, COLUMNS="400", **env),
                         capture_output=True, text=True)
    if log_dir:
        with open(os.path.join(log_dir, f"mutant{number}_{tag}.log"), "w") as f:
            f.write(res.stdout[-20000:] + res.stderr[-5000:])
    if res.returncode == 0:
        return "survived"
    summary = [ln for ln in res.stdout.splitlines() if ln.startswith(("FAILED ", "ERROR "))]
    if res.returncode != 1 or len(summary) != 1 or not summary[0].startswith("FAILED "):
        raise SystemExit(f"mutant {number}: pytest ended with {res.returncode} and no single "
                         f"failed test\n{res.stdout[-3000:]}{res.stderr[-3000:]}")
    return "killed by " + summary[0].split(" - ")[0][len("FAILED tests/"):]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--dry-run", action="store_true", help="edit and compile only")
    ap.add_argument("--only", type=int, nargs="*", help="mutant numbers (default: all)")
    ap.add_argument("--logs", help="directory for each run's pytest output")
    ap.add_argument("--new-only", action="store_true", help="run only the new tests")
    args = ap.parse_args()
    if args.logs:
        os.makedirs(args.logs, exist_ok=True)
    B.build()     # the real library, whose objects the kernel mutants share
    rows = []
    for number, what, equivalent, edits in MUTANTS:
        if args.only and number not in args.only:
            continue
        host = edits[0][0] == "engine.py"
        tmp = tempfile.mkdtemp(prefix="mrx_poly_mutant_")
        try:
            if host:
                cwd, env = host_tree(tmp, edits), {}
                if args.dry_run:     # the copy imports and collects
                    subprocess.run([sys.executable, "-m", "pytest", "-q", "--collect-only",
                                    "-p", "no:cacheprovider", *NEW_TESTS, *OLD_TESTS], cwd=cwd,
                                   check=True, capture_output=True)
            else:
                csrc = ME.mutate(tmp, [])
                apply(os.path.join(csrc, P), edits)
                assert os.path.exists(ME.build_mutant(number, csrc))
                cwd, env = ROOT, {"MRX_LIB": f"libmrx_mutant{number}.so"}
            if args.dry_run:
                row = (number, what, "built", "built")
            else:
                row = (number, what, run_tests(NEW_TESTS, cwd, env, "new", number, args.logs),
                       "not run" if args.new_only else
                       run_tests(OLD_TESTS, cwd, env, "old", number, args.logs))
            rows.append(row + ("equivalent (argued)" if equivalent else "",))
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
            if not host:
                ME.remove_mutant(number)
        print("| {} | {} | {} | {} | {} |".format(*rows[-1]), flush=True)
    print("\n| # | mutant | new tests | old tests | note |\n|---|---|---|---|---|")
    for row in rows:
        print("| {} | {} | {} | {} | {} |".format(*row))
    survivors = [r[0] for r in rows if r[2] == "survived" and not r[4]]
    if survivors:
        raise SystemExit(f"the new tests let mutants {survivors} live")


if __name__ == "__main__":
    main()
