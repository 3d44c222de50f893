"""Developer tool: per-phase cycle totals of the team kernel.  Build and run:
    MRX_NVCC_FLAGS="-DMRX_DEV -DMRX_TEAM_PROFILE" MRX_LIB_NAME=libmrx_prof.so python -m matterport_maskrcnn_with_tensorflow_serving_b200.build
    MRX_LIB=libmrx_prof.so MRX_EXPAND_TEAMS=6x5x10 python tools/team_profile.py  Prints mean cycles per tile for warp 0 of a team and for
the other warps."""
import ctypes
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from matterport_maskrcnn_with_tensorflow_serving_b200 import synth, _native  # noqa: E402
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import UnmoldEngine, make_geom  # noqa: E402

teams, warps, rows = [int(v) for v in os.environ.get("MRX_EXPAND_TEAMS", "6x5x10").split("x")]
COCO = "--coco" in sys.argv   # BASELINE configs[2] instead: 64 x 800x1333, 1-100 instances each
if COCO:
    ims = synth.make_batch(7, 64, (800, 1333), (1, 100), num_classes=81)
else:
    ims = synth.make_batch(20260921, 32, (1024, 1024), 100, num_classes=81)
d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
eng = UnmoldEngine(len(ims), 100, (28, 28), 81)
eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims])
for _ in range(3):
    eng.enqueue(d_det, d_msk)
torch.cuda.synchronize()
lib = _native.load()
SLOTS = 256   # kProfCtas of csrc/expand_team.cu
sms = torch.cuda.get_device_properties(0).multi_processor_count
buf = np.zeros(SLOTS * 32 * 12, dtype=np.int64)
rc = lib.mrx_debug_team_profile(buf.ctypes.data_as(ctypes.c_void_p), buf.size)
assert rc == 0
a = buf.reshape(SLOTS, 32, 12)[:sms, :teams * warps].reshape(sms, teams, warps, 12).astype(np.float64)
tiles_per_team = 32 * (1024 // rows + (1 if 1024 % rows else 0)) * 32 / (sms * teams)
if COCO:
    tiles_per_team = 1.0   # (tile count depends on every image's N: totals per team instead)
names = ["B2 wait", "zero", "B3 wait", "items", "fence+B1 wait", "post-B1 (cull | store+decode+drain)", "w0: store issue", "w0: decode"]
print("mean cycles per tile (tiles/team = %.1f)" % tiles_per_team)
for k, nm in enumerate(names):
    w0 = a[:, :, 0, k].mean() / tiles_per_team
    ot = a[:, :, 1:, k].mean() / tiles_per_team
    mx = a[:, :, 1:, k].max(axis=2).mean() / tiles_per_team
    print(f"  {nm:40s} warp0 {w0:9.0f}   others mean {ot:9.0f}   others max-warp {mx:9.0f}")
tot = a[:, :, :, :6].sum(axis=3).mean() / tiles_per_team
print("  total per tile: %.0f cycles" % tot)
items = a[..., 10].sum(); rows = a[..., 11].sum()
print("  fast-path items: %.0f (%.2f per tile), rows/item %.1f, setup cycles/item %.0f, row-loop cycles/item %.0f (%.1f per row)" % (
    items, items / (tiles_per_team * sms * teams), rows / items, a[..., 8].sum() / items, a[..., 9].sum() / items, a[..., 9].sum() / rows))
