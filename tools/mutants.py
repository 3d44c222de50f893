"""The harness of the tools/mutate_<suite>.py scripts.  A mutant is a small, wrong edit of the
sources; the harness builds each one and reports which tests notice it.  A suite module defines:

    NEW_TESTS, OLD_TESTS   the pytest selections each mutant runs under (new, then old)
    DESELECT               test ids left out of every run
    EQUIVALENT             numbers of the mutants no input can tell from the correct code
    MUTANTS                (number, what it models, [(file, old, new, count)]), or with a fourth
                           element (new, old) that replaces the suite's selections for that
                           mutant; a selection of None is not run

An edit replaces `old` by `new` in `file`, a package .py file or a csrc/ file; a pattern found
other than `count` times is an error.  Kernel mutants (csrc/ edits) are applied to a temporary
copy of csrc/ and include/, built as lib/libmrx_mutant<n>.so through build.py's MRX_LIB_NAME
hook and selected with MRX_LIB.  Host mutants (.py edits) run on a temporary copy of the package
and tests/, with the real library, include/ and oracle/ linked in.  A mutant does not mix the
two.  Each selection runs once, in a subprocess, stopping at its first failure, and ends in one
verdict:

    survived   pytest exits 0
    killed     pytest exits 1 with exactly one FAILED summary line and no ERROR line; reported
               as `killed by <test> (<exception name>)`
    fault      a FAILED or ERROR line reports a CUDA error (torch's `CUDA error:`, or an MrxError
               with status MRX_E_CUDA): a finding to explain, not a kill.  The script prints the
               log's tail and stops; the mutant is not run again
    no verdict any other ending (a collection or fixture error, a usage error, a crash): the
               script stops

The temporary copy and the mutant library are removed after each mutant; the repository's
sources and build are not touched.  The script exits non-zero when a mutant that is not
equivalent survives the new tests.  Development scripts: only tests/test_host_mutants.py, which
checks the tables on the CPU, imports them."""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from matterport_maskrcnn_with_tensorflow_serving_b200 import _native  # noqa: E402
from matterport_maskrcnn_with_tensorflow_serving_b200 import build as B  # noqa: E402

PKG = os.path.basename(B.PKG_DIR)


def source(root, file):
    """Where `file`, as an edit names it, lies in a tree rooted at `root`."""
    pkg = os.path.join(root, PKG)
    return os.path.join(pkg, file) if file.endswith(".py") else os.path.join(pkg, "csrc", file)


def is_host(edits):
    kinds = {file.endswith(".py") for file, _, _, _ in edits}
    if len(kinds) != 1:
        raise SystemExit(f"a mutant edits kernel sources or package .py files, not both: {edits}")
    return kinds.pop()


def edited(root, edits):
    """{path: text} of the files under `root` that `edits` touch, the edits applied in order."""
    texts = {}
    for file, old, new, count in edits:
        path = source(root, file)
        if path not in texts:
            with open(path) as f:
                texts[path] = f.read()
        found = texts[path].count(old)
        if found != count:
            raise SystemExit(f"{file}: pattern found {found} times, not {count}: {old!r}")
        texts[path] = texts[path].replace(old, new)
    return texts


def selections(suite, mutant):
    """(new, old) pytest selections of a mutant."""
    return mutant[3] if len(mutant) > 3 else (suite.NEW_TESTS, suite.OLD_TESTS)


def copy_tree(tmp, host):
    """The sources under `tmp`, laid out as in the repository (common.cuh includes
    ../../include/mrx.h).  Host: the package with lib/ linked to the real build, tests/, and
    links to include/ and oracle/.  Kernel: csrc/ and include/."""
    if host:
        pkg = os.path.join(tmp, PKG)
        shutil.copytree(B.PKG_DIR, pkg, ignore=shutil.ignore_patterns("lib", "__pycache__"))
        os.symlink(B.LIB_DIR, os.path.join(pkg, "lib"))
        shutil.copytree(os.path.join(ROOT, "tests"), os.path.join(tmp, "tests"),
                        ignore=shutil.ignore_patterns("__pycache__"))
        for name in ("include", "oracle"):
            os.symlink(os.path.join(ROOT, name), os.path.join(tmp, name))
    else:
        shutil.copytree(B.CSRC, os.path.join(tmp, PKG, "csrc"))
        shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))


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


def is_fault(line):
    return "CUDA error" in line or "MrxError" in line and f"(status {_native.MRX_E_CUDA})" in line


def verdict(number, tag, selection, deselect, cwd, env, log_dir):
    """The verdict of one selection's run (module docstring); 'not run' for a None selection."""
    if selection is None:
        return "not run"
    # COLUMNS: pytest cuts the summary lines read below to the terminal's width
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-rfE", "-p", "no:cacheprovider",
           *selection, *(a for t in deselect for a in ("--deselect", t))]
    res = subprocess.run(cmd, cwd=cwd, env=dict(os.environ, COLUMNS="400", **env),
                         capture_output=True, text=True)
    if log_dir:
        with open(os.path.join(log_dir, f"mutant{number}_{tag}.log"), "w") as f:
            f.write(res.stdout[-20000:] + res.stderr[-5000:])
    if res.returncode == 0:
        return "survived"
    tail = res.stdout[-3000:] + res.stderr[-3000:]
    summary = [ln for ln in res.stdout.splitlines() if ln.startswith(("FAILED ", "ERROR "))]
    if any(is_fault(ln) for ln in summary):
        raise SystemExit(f"mutant {number}: a CUDA error under the {tag} tests, a fault and not "
                         f"a kill\n{tail}")
    if res.returncode != 1 or len(summary) != 1 or not summary[0].startswith("FAILED "):
        raise SystemExit(f"mutant {number}: pytest ended with {res.returncode} and no single "
                         f"failed test\n{tail}")
    test, _, message = summary[0][len("FAILED tests/"):].partition(" - ")
    # pytest shows a failed `assert` as the statement, any other exception as `<type>: <text>`
    exception = "AssertionError" if message.startswith("assert ") else \
        message.split(":")[0].rsplit(".", 1)[-1]
    return f"killed by {test} ({exception})"


def main(suite):
    ap = argparse.ArgumentParser(description=suite.__doc__.split("\n\n")[0])
    ap.add_argument("--dry-run", action="store_true",
                    help="edit and compile only (host mutants: collect the tests)")
    ap.add_argument("--only", type=int, nargs="*", help="mutant numbers (default: all)")
    ap.add_argument("--logs", help="directory for each run's pytest output")
    ap.add_argument("--new-only", action="store_true",
                    help="run only the new tests (the older ones can take minutes per mutant)")
    ap.add_argument("--old-only", action="store_true", help="run only the older tests")
    args = ap.parse_args()
    if args.logs:
        os.makedirs(args.logs, exist_ok=True)
    B.build()     # the real library, whose objects the kernel mutants share
    rows = []
    for mutant in suite.MUTANTS:
        number, what, edits = mutant[:3]
        if args.only and number not in args.only:
            continue
        new, old = selections(suite, mutant)
        host = is_host(edits)
        tmp = tempfile.mkdtemp(prefix="mrx_mutant_")
        try:
            copy_tree(tmp, host)
            for path, text in edited(tmp, edits).items():
                with open(path, "w") as f:
                    f.write(text)
            if host:
                cwd, env = tmp, {}
                if args.dry_run:     # the copy imports and collects
                    subprocess.run([sys.executable, "-m", "pytest", "-q", "--collect-only",
                                    "-p", "no:cacheprovider", *new, *(old or [])], cwd=cwd,
                                   check=True, capture_output=True)
            else:
                assert os.path.exists(build_mutant(number, os.path.join(tmp, PKG, "csrc")))
                cwd, env = ROOT, {"MRX_LIB": f"libmrx_mutant{number}.so"}
            if args.dry_run:
                row = [number, what] + ["collected" if host else "built"] * 2
            else:
                row = [number, what,
                       "not run" if args.old_only else
                       verdict(number, "new", new, suite.DESELECT, cwd, env, args.logs),
                       "not run" if args.new_only else
                       verdict(number, "old", old, suite.DESELECT, cwd, env, args.logs)]
            rows.append(row + ["equivalent (argued)" if number in suite.EQUIVALENT else ""])
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
            remove_mutant(number)
        print("| {} | {} | {} | {} | {} |".format(*rows[-1]), flush=True)
    print("\n| # | mutant | new tests | old tests | note |\n|---|---|---|---|---|")
    for row in rows:
        print("| {} | {} | {} | {} | {} |".format(*row))
    survivors = [r[0] for r in rows if r[2] == "survived" and r[0] not in suite.EQUIVALENT]
    if survivors:
        raise SystemExit(f"the new tests let mutants {survivors} live")
