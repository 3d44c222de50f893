"""Run every kernel of the library once or twice so that one ncu invocation can capture them:

  ncu --set full --clock-control none --import-source on -k regex:'<names>' -o build/aux \
      python tools/profile_aux.py [--batch 32]

Kernels launched (in this order, after one warm-up pass): unmold_prologue, gather_tiles,
mask_expand_team, mask_expand_bits (packed output), pack_masks, composite_masks, anchors,
cv2_resize (single + batch), mold_image (three source sizes + batch)."""
import argparse
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from matterport_maskrcnn_with_tensorflow_serving_b200 import synth, visualize  # noqa: E402
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import (  # noqa: E402
    AnchorGenerator, Molder, UnmoldEngine, make_geom)
from matterport_maskrcnn_with_tensorflow_serving_b200.model_configs import MaskRCNNServingConfig  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--coco", action="store_true",
                help="BASELINE configs[2] instead: 800x1333 images, 1-100 instances each")
args = ap.parse_args()
torch.cuda.set_device(0)
if args.coco:
    ims = synth.make_batch(7, args.batch, (800, 1333), (1, 100), num_classes=81)
else:
    ims = bench.make_bench_images(0, args.batch)
d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
eng = UnmoldEngine(args.batch, 100, (28, 28), 81)
eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims])
gen = AnchorGenerator(MaskRCNNServingConfig)
m = Molder(MaskRCNNServingConfig)
rng = np.random.default_rng(0)
big = synth.synth_rgb_image(rng, 1080, 1920)
d_big = torch.from_numpy(big).cuda()
srcs = [torch.from_numpy(synth.synth_rgb_image(rng, *hw)).cuda()
        for hw in [(1024, 1024), (800, 1333), (2160, 3840)]]
img = torch.from_numpy(synth.synth_rgb_image(rng, *ims[0].original_image_shape[:2])).cuda()
colors = visualize.random_colors(100, rng=random.Random(0))
for _ in range(2):
    eng.enqueue(d_det, d_msk)
    eng.enqueue_expand_packed()
    eng.pack_masks()
    visualize.composite_batch(eng, [img] * args.batch, colors)
    gen.generate_device((1024, 1024, 3))
    m.cv2_resize_device(d_big, (640, 640))
    d640 = m.cv2_resize_batch_device([big] * 8, (640, 640))
    for s in srcs:
        m.mold_device(s, np.float32)
    m.mold_batch_device(d640, np.float32)
torch.cuda.synchronize()
