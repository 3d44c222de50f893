"""Repeat-launch stress of the team expand kernel: its teams of warps synchronise through named
barriers, hand out tiles from a global ticket counter and drain each tile buffer with bulk copies
before re-zeroing it, so a protocol bug shows up as a rare hang or as a byte that differs between
launches.  Runs a few hundred launches over mixed shapes and checks every result against the
first one (the output is a pure function of the inputs: a team only ever stores 1s into a tile
buffer it has zeroed)."""
import numpy as np
import pytest

from matterport_maskrcnn_with_tensorflow_serving_b200 import synth
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import UnmoldEngine, make_geom

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


@pytest.mark.parametrize("hw,n,batch,chunk", [
    ((1024, 1024), 100, 8, 0),          # strip units, default chunk
    ((1024, 1024), 100, 8, 51200),      # fewer, larger chunk buffers
    ((800, 1333), (1, 100), 6, 0),      # flat units, ragged counts
    ((96, 160), (0, 16), 40, 4096),     # many tiny images, tiny chunks, empty images
])
def test_repeat_launches_are_identical(cuda_device, hw, n, batch, chunk):
    import torch

    R = 100 if hw[0] >= 800 else 16
    ims = synth.make_batch(91, batch, hw, n, num_classes=7, max_instances=R)
    eng = UnmoldEngine(batch, R, (28, 28), 7, chunk_bytes=chunk)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims])
    d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
    eng.enqueue(d_det, d_msk)
    torch.cuda.synchronize()
    counts = eng.d_counts[:batch].cpu().numpy()
    total = int(eng._offsets[batch])
    ref = eng.d_canvas[:total].clone()
    ref_sum = int(ref.sum(dtype=torch.int64))
    assert ref_sum > 0 or int(counts.sum()) == 0
    launches = 150
    for it in range(launches):
        eng.d_canvas[:total].fill_(7)            # poison: every byte must be rewritten
        eng.enqueue(d_det, d_msk)
        if it % 25 == 24:
            torch.cuda.synchronize()
            # bytes inside each image's [H,W,N_b] prefix must match; the tail of a slot
            # (capacity H*W*R) is not part of the result
            for b in range(batch):
                o = int(eng._offsets[b])
                k = int(counts[b]) * hw[0] * hw[1]
                assert torch.equal(eng.d_canvas[o:o + k], ref[o:o + k]), (it, b)
    torch.cuda.synchronize()
