"""The mutant tables of tools/mutate_<suite>.py, checked on the CPU: every edit still finds its
pattern in today's sources exactly as often as it states, so a change that moves an edited line
fails here instead of on the suite's next GPU run; and every test a table names exists."""
import importlib
import os
import re
import sys
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mutants  # noqa: E402

SUITES = ["expand", "eval", "preprocess", "polygons", "jpeg", "png_decode", "png_encode", "contours"]


def check_table(suite, root):
    numbers = [mutant[0] for mutant in suite.MUTANTS]
    assert len(set(numbers)) == len(numbers), f"mutant numbers repeat: {numbers}"
    assert set(suite.EQUIVALENT) <= set(numbers), f"EQUIVALENT {suite.EQUIVALENT} names no mutant"
    tests = set(suite.DESELECT)
    for mutant in suite.MUTANTS:
        number, _, edits = mutant[:3]
        assert all(old != new for _, old, new, _ in edits), f"mutant {number} edits nothing"
        mutants.is_host(edits)
        mutants.edited(root, edits)     # SystemExit when a pattern's count is off
        for selection in mutants.selections(suite, mutant):
            tests.update(selection or [])
    for test in tests:
        path, _, name = test.partition("::")
        assert os.path.isfile(os.path.join(root, path)), f"{test}: no such file"
        if name:
            with open(os.path.join(root, path)) as f:
                assert re.search(rf"^def {re.escape(name)}\(", f.read(), re.M), \
                    f"{test}: no such test"


@pytest.mark.parametrize("name", SUITES)
def test_table_matches_the_sources(name):
    check_table(importlib.import_module(f"mutate_{name}"), ROOT)


def _table(**change):
    fields = dict(NEW_TESTS=["tests/test_a.py"], OLD_TESTS=["tests/test_b.py"],
                  DESELECT=["tests/test_b.py::test_slow"], EQUIVALENT={1},
                  MUTANTS=[(1, "k", [("k.cu", "a >= b", "a > b", 2)]),
                           (2, "host", [("engine.py", "x + 1", "x + 2", 1)])])
    fields.update(change)
    return types.SimpleNamespace(**fields)


@pytest.fixture
def tree(tmp_path):
    """A root holding k.cu (`a >= b` twice), engine.py and two test files."""
    pkg = tmp_path / mutants.PKG
    (pkg / "csrc").mkdir(parents=True)
    (pkg / "csrc" / "k.cu").write_text("if (a >= b) x;\nif (a >= b) y;\n")
    (pkg / "engine.py").write_text("y = x + 1\n")
    (tmp_path / "tests").mkdir()
    (tmp_path / "tests" / "test_a.py").write_text("def test_one():\n    pass\n")
    (tmp_path / "tests" / "test_b.py").write_text("def test_slow():\n    pass\n")
    return str(tmp_path)


def test_synthetic_table_passes(tree):
    check_table(_table(), tree)


@pytest.mark.parametrize("change, error", [
    (dict(MUTANTS=[(1, "k", [("k.cu", "a >= b", "a > b", 1)])]), "found 2 times, not 1"),
    (dict(MUTANTS=[(1, "k", [("k.cu", "a > b", "a >= b", 1)])]), "found 0 times, not 1"),
    (dict(MUTANTS=[(1, "k", [("k.cu", "a >= b", "a >= b", 2)])]), "edits nothing"),
    (dict(MUTANTS=[(1, "k", [("k.cu", "a >= b", "a > b", 2)]),
                   (1, "k", [("k.cu", "a >= b", "a < b", 2)])]), "numbers repeat"),
    (dict(EQUIVALENT={3}), "names no mutant"),
    (dict(MUTANTS=[(1, "both", [("k.cu", "a >= b", "a > b", 2),
                                ("engine.py", "x + 1", "x + 2", 1)])]), "not both"),
    (dict(OLD_TESTS=["tests/test_c.py"]), "no such file"),
    (dict(DESELECT=["tests/test_b.py::test_fast"]), "no such test"),
    (dict(MUTANTS=[(1, "k", [("k.cu", "a >= b", "a > b", 2)],
                    (["tests/test_a.py::test_two"], None))]), "no such test"),
])
def test_broken_table_fails(tree, change, error):
    with pytest.raises((AssertionError, SystemExit), match=error):
        check_table(_table(**change), tree)
