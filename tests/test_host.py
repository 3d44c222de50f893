"""CPU tests of the host side: the C-ABI library loads and exports every symbol that
include/mrx.h declares (no compute calls without a GPU), argument validation that does not
need a device, host geometry logic vs the oracle, the product path refuses to run without
CUDA, image sharding, and the gather plumbing under gloo with world_size 2."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N
from matterport_maskrcnn_with_tensorflow_serving_b200 import serve, sharding, synth
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import make_geom, resize_image_geometry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    lib = N.load()
    declared = N.declared_symbols()
    assert len(declared) >= 10
    assert sorted(N.SIGNATURES) == declared          # the binding covers the whole header
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.mrx_abi_version() == N.ABI_VERSION


def test_host_side_argument_validation():
    lib = N.load()
    out = C.c_longlong(0)
    strides = N.int_array([4, 8, 16, 32, 64])
    assert lib.mrx_anchor_count(1024, 1024, strides, 5, 3, 1, C.byref(out)) == 0
    assert out.value == 261888
    assert lib.mrx_anchor_count(1030, 770, strides, 5, 3, 2, C.byref(out)) == 0
    want = 3 * sum(-(-(-(-1030 // s)) // 2) * -(-(-(-770 // s)) // 2) for s in (4, 8, 16, 32, 64))
    assert out.value == want
    assert lib.mrx_anchor_count(1024, 1024, strides, 9, 3, 1, C.byref(out)) == -2     # > MRX_MAX_LEVELS
    assert b"n_levels" in lib.mrx_last_error()
    assert lib.mrx_anchors(None, 1024, 1024, None, None, strides, 5, 3, 1, None) == -1
    assert lib.mrx_mask_expand(None, None, None, None, None, None, None, 1, 100, 28, 28, 0,
                               0, None, None) == -1
    assert lib.mrx_mask_expand_values(None, None, None, None, None, None, None, None, 1, 100,
                                      28, 28, None, None) == -1
    p16 = C.c_void_p(16)
    assert lib.mrx_unmold_prepare(p16, 0, p16, 3, 1, 100, 28, 28, 81, p16, p16, p16, p16, p16,
                                  p16, p16, p16, p16, None) == -1      # bad mask dtype
    assert lib.mrx_peer_export(None, None) == -1 and lib.mrx_peer_wait(None, 1, 1, None) == -1


# The entry points that read a tile batch, as (tile_index, B, R, mh, mw) -> status; every other
# argument is a non-null placeholder.  The lane kernels keep a tile row in one warp's lanes.
def _tile_batch_entry_points(lib):
    p = C.c_void_p(16)
    return {
        "mrx_mask_expand": lambda ti, B, R, mh, mw: lib.mrx_mask_expand(
            p, ti, p, p, p, p, p, B, R, mh, mw, 0, 0, p, None),
        "mrx_mask_expand_values": lambda ti, B, R, mh, mw: lib.mrx_mask_expand_values(
            p, ti, p, p, p, p, p, p, B, R, mh, mw, p, None),
        "mrx_mask_expand_packed": lambda ti, B, R, mh, mw: lib.mrx_mask_expand_packed(
            p, ti, p, p, p, p, p, B, R, mh, mw, 1024, p, None),
        "mrx_rle_count": lambda ti, B, R, mh, mw: lib.mrx_rle_count(
            p, ti, p, p, p, p, p, B, R, mh, mw, 1024, None),
        "mrx_rle_write": lambda ti, B, R, mh, mw: lib.mrx_rle_write(
            p, ti, p, p, p, p, p, p, p, B, R, mh, mw, 1024, None),
    }


# (what is wrong, null tile index, B, R, mh, mw, status, lane kernels only)
BAD_TILE_BATCHES = [
    ("B > MRX_MAX_BATCH", False, N.MRX_MAX_BATCH + 1, 100, 28, 28, -1, False),
    ("R = 0", False, 1, 0, 28, 28, -1, False),
    ("R = 65535", False, 1, 65535, 28, 28, -1, False),
    ("mh = 1", False, 1, 100, 1, 28, -2, False),
    ("mw % 4 != 0", False, 1, 100, 28, 6, -2, False),
    ("mw > MRX_MAX_LANE_MASK_W", False, 1, 100, 28, 32, -2, True),
    ("null tile index", True, 1, 100, 28, 28, -1, False),
]


@pytest.mark.parametrize("fn", ["mrx_mask_expand", "mrx_mask_expand_values",
                                "mrx_mask_expand_packed", "mrx_rle_count", "mrx_rle_write"])
def test_tile_batch_checks_agree(fn):
    """Every entry point that reads the tile batch refuses the same bad inputs with the same
    status, names itself in the message, and returns before touching the device."""
    lib = N.load()
    call = _tile_batch_entry_points(lib)[fn]
    lane = fn != "mrx_mask_expand"
    for what, null_index, B, R, mh, mw, status, lane_only in BAD_TILE_BATCHES:
        if lane_only and not lane:
            continue
        assert call(None if null_index else C.c_void_p(16), B, R, mh, mw) == status, what
        msg = lib.mrx_last_error().decode()
        assert msg.startswith(fn + ":"), (what, msg)
        if status == -2:
            limit = N.MRX_MAX_LANE_MASK_W if lane else N.MRX_MAX_MASK_DIM
            assert f"mw<={limit}" in msg, (what, msg)


def test_product_path_has_no_cpu_fallback():
    import torch

    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils

    im = synth.make_batch(0, 1, (64, 64), 2, num_classes=3)[0]
    with pytest.raises(N.MrxError):
        api_utils.unmold_detections(im.detections, im.mrcnn_mask, im.original_image_shape,
                                    im.image_shape, im.window)
    with pytest.raises(N.MrxError):
        api_utils.get_anchors((64, 64, 3))


def test_product_does_not_import_the_oracle():
    pkg = os.path.join(ROOT, "matterport_maskrcnn_with_tensorflow_serving_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text, f


@pytest.mark.parametrize("hw", [(1024, 1024), (800, 1333), (2160, 3840), (480, 640), (100, 37)])
@pytest.mark.parametrize("mode", ["square", "pad64", "none"])
def test_resize_image_geometry_matches_oracle(hw, mode):
    if mode == "pad64" and max(hw) > 1024:
        pytest.skip("pad64 keeps the scaled size; covered by the smaller shapes")
    img = np.zeros((hw[0], hw[1], 3), dtype=np.uint8)
    kw = dict(min_dim=128 if mode == "pad64" else 800, max_dim=1024, min_scale=0, mode=mode)
    ref, window, scale, padding, crop = oracle.resize_image(img, **kw)
    nh, nw, top, left, oh, ow, win, sc, pad = resize_image_geometry(
        hw[0], hw[1], kw["min_dim"], kw["max_dim"], kw["min_scale"], mode)
    assert (oh, ow) == ref.shape[:2] and win == window and sc == scale and pad == padding


def test_compose_image_meta_and_geom():
    meta = serve.compose_image_meta(0, (640, 640, 3), (1024, 1024, 3), (112, 112, 912, 912), 1.25,
                                    np.zeros(81, np.int32))
    ref = oracle.compose_image_meta(0, (640, 640, 3), (1024, 1024, 3), (112, 112, 912, 912), 1.25,
                                    np.zeros(81, np.int32))
    np.testing.assert_array_equal(meta, ref)
    assert make_geom((800, 1333, 3), (1024, 1024, 3), (204, 0, 819, 1024)) == \
        [800, 1333, 1024, 1024, 204, 0, 819, 1024]


def test_synth_inputs_are_valid_for_the_reference():
    ims = synth.make_batch(9, 3, (800, 1333), (1, 100))
    for im in ims:
        b, c, s, m = oracle.unmold_detections(im.detections.astype(np.float64),
                                              im.mrcnn_mask[:, :, :, :].astype(np.float64),
                                              im.original_image_shape, im.image_shape, im.window)
        assert b.shape[0] == im.n_valid                     # nothing dropped, nothing out of canvas
        assert (b[:, 0] >= 0).all() and (b[:, 2] <= 800).all() and (b[:, 3] <= 1333).all()
        assert (c >= 1).all()
        assert (im.mrcnn_mask.reshape(100, -1, 81).min(axis=1) < 0.5).all()   # SURVEY 8c corner case


# ------------------------------------------------------------------ sharding
def test_partition_images_contiguous_and_balanced():
    costs = [100] * 128
    parts = sharding.partition_images(costs, 8)
    assert parts == [(16 * r, 16 * (r + 1)) for r in range(8)]
    rng = np.random.default_rng(0)
    costs = rng.integers(1, 101, size=64) * 800 * 1333          # config 3: ragged instance counts
    parts = sharding.partition_images(costs, 8)
    assert parts[0][0] == 0 and parts[-1][1] == 64
    assert all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
    loads = [costs[a:b].sum() for a, b in parts]
    assert max(loads) <= 1.35 * (costs.sum() / 8)
    assert sharding.partition_images([], 4) == [(0, 0)] * 4
    assert sharding.partition_images([5, 5], 4)[-1][1] == 2
    assert sharding.equal_partition(10, 3) in ([(0, 3), (3, 7), (7, 10)], [(0, 3), (3, 6), (6, 10)],
                                               [(0, 4), (4, 7), (7, 10)])


def test_chunk_splits():
    assert sharding.chunk_bounds(16, 4) == [(0, 4), (4, 8), (8, 12), (12, 16)]
    assert sharding.chunk_bounds(3, 8) == [(0, 1), (1, 2), (2, 3)]
    assert sharding.chunk_bounds(0, 4) == []
    for size, n in [(1000, 4), (17, 4), (0, 3), (3355443200, 7), (16, 1)]:
        r = sharding.RootGather.chunk_ranges(size, n)
        assert len(r) == n and r[0][0] == 0 and r[-1][1] == size
        assert all(a[1] == b[0] for a, b in zip(r, r[1:]))
        assert all(lo % 16 == 0 for lo, _ in r)


_GLOO_WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from matterport_maskrcnn_with_tensorflow_serving_b200 import sharding
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:" + sys.argv[2],
                        rank=int(sys.argv[3]), world_size=2)
rank = dist.get_rank()
costs = [7, 3, 5, 9, 1]                      # bytes per image (stand-in canvases)
parts = sharding.partition_images(costs, 2)
lo, hi = parts[rank]
local = torch.cat([torch.full((costs[i],), 10 * i + 1, dtype=torch.uint8) for i in range(lo, hi)]) \
    if hi > lo else torch.empty(0, dtype=torch.uint8)
sizes = [sum(costs[a:b]) for a, b in parts]
out = sharding.gather_bytes_to_root(local, sizes, 0)
want = np.concatenate([np.full(costs[i], 10 * i + 1, np.uint8) for i in range(len(costs))])
if rank == 0:
    got = torch.cat(out).numpy()
    assert np.array_equal(got, want), (got, want)
    print("GATHER_OK", parts)
else:
    assert out is None
# pipelined gather into one preallocated buffer, several chunks per rank, used twice
big = [4000 + 37, 2500 + 3]
src = [torch.arange(big[r], dtype=torch.int64).mul(7 + r).remainder(251).to(torch.uint8) for r in range(2)]
g = sharding.RootGather(big, "cpu")
for rep in range(2):
    mine = (src[rank] + rep).to(torch.uint8)
    n_chunks = 3
    g.begin(n_chunks)
    if rank == 0:
        g.slot(0).copy_(mine)                 # rank 0's kernels write straight into its slot
        for _ in range(n_chunks):
            g.post()
    else:
        for lo, hi in sharding.RootGather.chunk_ranges(big[rank], n_chunks):
            g.post(mine, lo, hi)
    g.wait()
    if rank == 0:
        for r in range(2):
            assert torch.equal(g.slot(r), (src[r] + rep).to(torch.uint8)), (rep, r)
        assert g.recv.numel() == sum(big)
    dist.barrier()
if rank == 0:
    print("PIPELINED_OK")
dist.barrier()
dist.destroy_process_group()
'''


def test_gather_to_root_gloo_world_size_2(tmp_path):
    script = tmp_path / "gloo_worker.py"
    script.write_text(_GLOO_WORKER)
    port = str(29500 + (os.getpid() % 2000))
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, port, str(r)],
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for r in range(2)]
    outs = [p.communicate(timeout=240)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    assert "GATHER_OK" in outs[0] and "PIPELINED_OK" in outs[0]


def test_dropin_shims_resolve_the_reference_imports():
    """serve.py:21-23 import lines work against dropin/ (run in a clean interpreter)."""
    code = ("import sys; sys.path.insert(0, %r);"
            "from api.helpers import utils as api_utils; import configs as cf;"
            "from model_configs import mconfig as mcf;"
            "assert callable(api_utils.get_anchors) and callable(api_utils.unmold_detections);"
            "assert callable(api_utils.load_img);"
            "assert cf.OUT_DETECTION_SHAPE == (100, 6) and mcf.IMAGE_MAX_DIM == 1024;"
            "print('ok')") % os.path.join(ROOT, "dropin")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr


def test_overlay_host_logic_matches_oracle():
    """visualize.random_colors / blend_table: the colour values and the float64 evaluation
    order `alpha * color[c] * 255` the reference's apply_mask uses (no GPU needed)."""
    import random

    from matterport_maskrcnn_with_tensorflow_serving_b200 import visualize

    assert visualize.random_colors(11, rng=random.Random(2)) == oracle.random_colors(11, rng=random.Random(2))
    assert visualize.random_colors(5, bright=False, rng=random.Random(0)) == \
        oracle.random_colors(5, bright=False, rng=random.Random(0))
    cols = oracle.random_colors(7, rng=random.Random(9))
    tab = visualize.blend_table(cols, 0.3, 10)
    assert tab.shape == (10, 3) and tab.dtype == np.float64
    for i, col in enumerate(cols):
        for c in range(3):
            assert tab[i, c] == 0.3 * col[c] * 255
    assert not tab[7:].any()
    # without CUDA the product raises instead of falling back
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(N.MrxError):
            visualize.apply_masks(np.zeros((4, 4, 3), np.uint8), np.zeros((1, 4), np.int32),
                                  np.zeros((4, 4, 1), bool), cols)


def test_no_unbound_global_names_in_the_package():
    """Static check (the GPU paths cannot run here): every name a module loads is bound
    somewhere in it (import, def, class, assignment, argument) or is a builtin."""
    import ast
    import builtins

    pkg = os.path.join(ROOT, "matterport_maskrcnn_with_tensorflow_serving_b200")
    files = [os.path.join(pkg, f) for f in sorted(os.listdir(pkg)) if f.endswith(".py")]
    files += [os.path.join(ROOT, "bench.py"), os.path.join(ROOT, "__graft_entry__.py")]
    for path in files:
        tree = ast.parse(open(path).read())
        bound = set(dir(builtins)) | {"__file__", "__name__", "__doc__"}
        for node in ast.walk(tree):
            if isinstance(node, (ast.FunctionDef, ast.ClassDef, ast.AsyncFunctionDef)):
                bound.add(node.name)
            elif isinstance(node, ast.arg):
                bound.add(node.arg)
            elif isinstance(node, (ast.Import, ast.ImportFrom)):
                for a in node.names:
                    bound.add((a.asname or a.name).split(".")[0])
            elif isinstance(node, ast.Name) and isinstance(node.ctx, (ast.Store, ast.Del)):
                bound.add(node.id)
            elif isinstance(node, ast.ExceptHandler) and node.name:
                bound.add(node.name)
        used = {n.id for n in ast.walk(tree) if isinstance(n, ast.Name) and isinstance(n.ctx, ast.Load)}
        assert not (used - bound), (os.path.basename(path), sorted(used - bound))


def test_bench_reference_arm_prints_one_json_line():
    """Contract of bench.py: rank 0's stdout carries exactly ONE line, the JSON result (library
    banners and worker output go to stderr).  The reference arm runs without a GPU."""
    import json
    import subprocess
    import sys
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference",
                          "--steps", "1", "--warmup", "0", "--cpu-procs", "2"],
                         capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, out.stdout
    line = json.loads(lines[0])
    assert line["impl"] == "reference" and line["metric"] == "instance-masks/sec"
    assert line["value"] > 0 and line["e2e"]["h2d_bytes_per_step"] == 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] == 2
