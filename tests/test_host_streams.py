"""CPU test of the package's stream rule (engine.py's module docstring): every libmrx call runs on
the current CUDA stream, and only the pipeline launches that streaming and sharding drive on
explicit streams take a `stream` argument, which does nothing but make that stream current
(`_native.on_stream`: torch.cuda.stream(stream) unless it is already current)."""
import ast
import os

import pytest

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                   "matterport_maskrcnn_with_tensorflow_serving_b200")

# (module, qualified name) of every function that takes `stream`
KEEP = {("engine", "UnmoldEngine.enqueue"), ("engine", "UnmoldEngine.enqueue_expand"),
        ("engine", "UnmoldEngine.enqueue_expand_packed"), ("engine", "UnmoldEngine.enqueue_packed"),
        ("sharding", "PeerGather.signal"), ("sharding", "PeerGather.wait"),
        ("_native", "stream_ptr"), ("_native", "on_stream")}
LAUNCHERS = sorted(KEEP - {("_native", "stream_ptr"), ("_native", "on_stream")})


def _modules():
    out = {}
    for name in sorted(os.listdir(PKG)):
        if name.endswith(".py"):
            with open(os.path.join(PKG, name)) as f:
                out[name[:-3]] = ast.parse(f.read(), name)
    return out


def _functions(modules):
    """(module, qualified name, node) of every function of the package."""
    out = []

    def walk(node, prefix, mod):
        for child in ast.iter_child_nodes(node):
            if isinstance(child, (ast.FunctionDef, ast.AsyncFunctionDef)):
                out.append((mod, prefix + child.name, child))
                walk(child, prefix + child.name + ".", mod)
            elif isinstance(child, ast.ClassDef):
                walk(child, prefix + child.name + ".", mod)

    for mod, tree in modules.items():
        walk(tree, "", mod)
    return out


MODULES = _modules()
FUNCTIONS = _functions(MODULES)


def _params(fn):
    a = fn.args
    return [p.arg for p in a.posonlyargs + a.args + a.kwonlyargs]


def test_only_the_pipeline_launches_take_a_stream():
    got = {(mod, q) for mod, q, fn in FUNCTIONS if "stream" in _params(fn)}
    assert got == KEEP, f"unexpected: {sorted(got - KEEP)}, missing: {sorted(KEEP - got)}"


@pytest.mark.parametrize("mod,qualname", LAUNCHERS)
def test_stream_only_makes_itself_current(mod, qualname):
    """The body names `stream` once: as the one argument of N.on_stream(...) in a `with`."""
    fn = next(f for m, q, f in FUNCTIONS if (m, q) == (mod, qualname))
    uses = [n for n in ast.walk(fn) if isinstance(n, ast.Name) and n.id == "stream"]
    assert len(uses) == 1, f"{qualname} names `stream` {len(uses)} times"
    ctx = [item.context_expr for w in ast.walk(fn) if isinstance(w, ast.With) for item in w.items]
    assert any(isinstance(c, ast.Call) and ast.unparse(c.func) == "N.on_stream"
               and len(c.args) == 1 and c.args[0] is uses[0] and not c.keywords for c in ctx), \
        f"{qualname}: `stream` is not on_stream's"


def test_every_launch_takes_the_current_stream():
    """No call of stream_ptr in the package passes an argument."""
    calls = [n for tree in MODULES.values() for n in ast.walk(tree) if isinstance(n, ast.Call)
             and (getattr(n.func, "attr", None) or getattr(n.func, "id", None)) == "stream_ptr"]
    assert len(calls) > 20
    passed = [(n.lineno, ast.unparse(n)) for n in calls if n.args or n.keywords]
    assert not passed, passed
