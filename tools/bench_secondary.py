"""Secondary workloads of BASELINE.json (configs[2], [3] per-GPU shard, [4]) and the mold step,
device-timed with CUDA events.  Not the contract bench (bench.py measures configs[1]); the
numbers go into README.md.  One JSON line per workload on stdout; the COCO compressed-RLE line of
each unmold workload also names the GPU and its power limit.

  python tools/bench_secondary.py [--iters 20] [--cpu]     (--cpu also times the oracle)
  python tools/bench_secondary.py --only-eval | --only-cocoeval | --only-bboxeval | --only-boundaryeval
                                  | --only-polygons | --only-lvis | --only-jpeg | --only-png
                                  | --only-jpeg-progressive | --only-png-decode | --only-jpeg-encode
                                  | --only-annotate
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from matterport_maskrcnn_with_tensorflow_serving_b200 import _native as N, synth  # noqa: E402
from matterport_maskrcnn_with_tensorflow_serving_b200.engine import (  # noqa: E402
    AnchorGenerator, Molder, UnmoldEngine, make_geom)
from matterport_maskrcnn_with_tensorflow_serving_b200.model_configs import MaskRCNNServingConfig  # noqa: E402


def time_ms(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(np.min(ts))


def unmold_case(name, batch, hw, n, classes, R, iters, base_images=4, seed=7, composite=False):
    base = synth.make_batch(seed, min(batch, base_images), hw, n, num_classes=classes, max_instances=R)
    ims = [base[i % len(base)] for i in range(batch)]
    d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
    eng = UnmoldEngine(batch, R, (28, 28), classes)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims])
    eng.enqueue(d_det, d_msk)
    torch.cuda.synchronize()
    counts = eng.d_counts[:batch].cpu().numpy()
    masks = int(counts.sum())
    out_bytes = eng.canvas_bytes(counts)
    algo = out_bytes + masks * (28 * 28 * 4 + 24)
    step_ms, _ = time_ms(lambda: eng.enqueue(d_det, d_msk), iters)

    k_ms, _ = time_ms(lambda: eng.enqueue_expand(), iters)
    # extension layout: the expand kernel that writes bit-packed masks, and the pack kernel
    pk_ms, _ = time_ms(lambda: eng.enqueue_expand_packed(), iters)
    pack_ms, _ = time_ms(lambda: eng.pack_masks(), iters)
    pro_ms, _ = time_ms(lambda: eng.enqueue(d_det, d_msk, expand=False), iters)
    # COCO RLE from the tiles (count pass, one host read of the totals, write pass)
    rle_ms, _ = time_ms(lambda: eng.enqueue_rle(), max(3, iters // 4))
    d_runs, off = eng.enqueue_rle()
    rle_bytes = int(d_runs.numel()) * 4
    strings = rle_strings_record(eng, d_runs, off, masks, iters)
    # contour polygons from the packed planes (count pass, one host read of the segment counts,
    # write pass, and the read of the contour counts): on planes already written, and with the
    # packed expand before it
    eng.enqueue_expand_packed()
    ct_ms, _ = time_ms(lambda: eng.trace_contours(), max(3, iters // 4))
    pct_ms, _ = time_ms(lambda: (eng.enqueue_expand_packed(), eng.trace_contours()), max(3, iters // 4))
    d_vert, d_coff, icoff = eng.trace_contours()
    n_vert, n_contours = int(d_vert.shape[0]), int(icoff[-1])
    contour_bytes = n_vert * 16 + (n_contours + 1) * 8 + icoff.size * 8
    if composite:
        import random

        from matterport_maskrcnn_with_tensorflow_serving_b200 import visualize
        rng = np.random.default_rng(1)
        images = [torch.from_numpy(synth.synth_rgb_image(rng, *hw)).cuda() for _ in range(min(batch, 2))]
        images = [images[i % len(images)] for i in range(batch)]
        colors = visualize.random_colors(R, rng=random.Random(0))
        c_ms, _ = time_ms(lambda: visualize.composite_batch(eng, images, colors), max(3, iters // 4))
        print(json.dumps({"workload": name + " -> mask overlay (display_instances blend) on the device canvas",
                          "composite_ms_incl_staging": round(c_ms, 3),
                          "canvas_read_GBps": round(out_bytes / c_ms / 1e6, 1),
                          "note": "includes the device-side staging copies of the 32 input images"}),
              flush=True)
    print(json.dumps({"workload": name, "images": batch, "hw": list(hw), "masks": masks,
                      "canvas_GB": round(out_bytes / 1e9, 3), "step_ms": round(step_ms, 4),
                      "Mmasks_per_s": round(masks / step_ms / 1e3, 3),
                      "expand_ms": round(k_ms, 4),
                      "expand_algorithmic_GBps": round(algo / k_ms / 1e6, 1),
                      "prologue_plus_class_gather_ms": round(pro_ms, 4),
                      "expand_packed_ms": round(pk_ms, 4),
                      "expand_packed_Mmasks_per_s": round(masks / pk_ms / 1e3, 2),
                      "rle_ms_incl_host_read": round(rle_ms, 4), "rle_output_MB": round(rle_bytes / 1e6, 2),
                      "contours_ms_incl_host_read": round(ct_ms, 4),
                      "expand_packed_plus_contours_ms": round(pct_ms, 4),
                      "contour_segments": n_vert - n_contours, "contours": n_contours,
                      "contour_vertices": n_vert, "contour_output_MB": round(contour_bytes / 1e6, 2),
                      "pack_kernel_ms": round(pack_ms, 4),
                      "pack_kernel_canvas_read_GBps": round(out_bytes / pack_ms / 1e6, 1)}), flush=True)
    print(json.dumps({"workload": name + " -> COCO compressed RLE strings", **strings, **card()}),
          flush=True)
    del eng, d_det, d_msk
    torch.cuda.empty_cache()


def card():
    """Name and power limit of the GPU the numbers come from (read-only nvidia-smi query)."""
    idx = (os.environ.get("CUDA_VISIBLE_DEVICES") or "0").split(",")[0]
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", idx], capture_output=True, text=True, timeout=60).stdout
        limit = float(out.strip())
    except (OSError, ValueError, subprocess.SubprocessError):
        limit = None
    return {"gpu": torch.cuda.get_device_name(0), "power_limit_W": limit}


def rle_strings_record(eng, d_runs, off, masks, iters):
    """mrx_rle_strings alone on the runs of the planned batch, and enqueue_rle_strings with the
    download of the strings; string bytes against the bytes of the kept instances' uint32 runs."""
    ni = eng._n_images * eng.R
    d_inst_off = torch.from_numpy(off).to(eng.device)
    d_str = torch.empty((N.rle_string_bound(off[-1], ni),), dtype=torch.uint8, device=eng.device)
    d_str_off = torch.empty((ni + 1,), dtype=torch.int64, device=eng.device)
    args = (d_runs, d_inst_off, eng.d_counts)

    def strings():
        N.check(eng.lib.mrx_rle_strings(*args, eng._n_images, eng.R, d_str_off, d_str,
                                        N.stream_ptr(None)), "mrx_rle_strings")

    def strings_downloaded():
        s, s_off = eng.enqueue_rle_strings()
        h_off = s_off.cpu().numpy()
        return s[:int(h_off[-1])].cpu().numpy()

    k_ms, _ = time_ms(strings, iters)
    e2e_ms, _ = time_ms(strings_downloaded, max(3, iters // 4))
    str_bytes = int(strings_downloaded().size)
    run_bytes = 4 * (int(off[-1]) + masks)      # T value changes -> T + masks runs
    return {"rle_strings_kernel_ms": round(k_ms, 4),
            "enqueue_rle_strings_ms_incl_download": round(e2e_ms, 4),
            "string_MB": round(str_bytes / 1e6, 3), "uncompressed_runs_MB": round(run_bytes / 1e6, 3),
            "string_over_runs": round(str_bytes / run_bytes, 4)}


def eval_case(iters, cpu):
    """configs[1] batch scored against ground truth: 32 x 1024x1024, 100 predictions against the
    100 instances of the same image jittered (synth.jitter_ground_truth).  The three kernels
    alone, and unmold_compute_ap_batch end to end (gt upload included) for one and for the ten
    thresholds of compute_ap_range, with the ground truth as bool masks and as COCO compressed
    strings (rle_gt_record); --cpu: the oracle's compute_overlaps_masks per image."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils
    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import mask_matches

    batch, base_n = 32, 4
    base = synth.make_batch(7, base_n, (1024, 1024), 100)
    rng = np.random.default_rng(8)
    jittered = [(j.detections, j.mrcnn_mask, j.original_image_shape, j.image_shape, j.window)
                for j in (synth.jitter_ground_truth(im, rng, 12, 0.1) for im in base)]
    base_gt = api_utils.unmold_detections_batch(jittered)
    # the same ground truth as COCO compressed strings, so that both paths score identical masks
    base_rle = [r[3] for r in api_utils.unmold_detections_rle_batch(jittered, compressed=True)]
    ims = [base[i % base_n] for i in range(batch)]
    gts = [(g[0], g[1], g[3]) for g in (base_gt[i % base_n] for i in range(batch))]
    items = [(im.detections, im.mrcnn_mask, im.original_image_shape, im.image_shape, im.window)
             for im in ims]
    eng = UnmoldEngine(batch, 100, (28, 28), 81)
    eng.plan([make_geom(im.original_image_shape, im.image_shape, im.window) for im in ims], canvas=False)
    d_det = torch.from_numpy(np.stack([im.detections for im in ims])).cuda()
    d_msk = torch.from_numpy(np.stack([im.mrcnn_mask for im in ims])).cuda()
    eng.enqueue_packed(d_det, d_msk)
    gt = eng.ground_truth([g[1] for g in gts], [g[2] for g in gts])
    d_ov = eng.enqueue_overlaps(gt)
    lib, n, R = eng.lib, batch, eng.R
    area_buf, ext_buf = eng._eval_bufs["areas"], eng._eval_bufs["extents"]

    def extents():
        N.check(lib.mrx_mask_extents(eng.d_packed, eng.d_packed_off, eng.d_counts, eng.d_geom,
                                     eng.d_boxes, area_buf, ext_buf, n, R, N.stream_ptr(None)),
                "mrx_mask_extents")

    ext_ms, _ = time_ms(extents, iters)
    ov_ms, _ = time_ms(lambda: eng.enqueue_overlaps(gt), iters)
    m1_ms, _ = time_ms(lambda: mask_matches(lib, d_ov, eng.d_counts, eng.d_class_ids, eng.d_scores,
                                            N.MRX_F32, gt, [0.5]), iters)
    thr10 = np.arange(0.5, 1.0, 0.05)
    m10_ms, _ = time_ms(lambda: mask_matches(lib, d_ov, eng.d_counts, eng.d_class_ids, eng.d_scores,
                                             N.MRX_F32, gt, thr10), iters)
    counts = eng.d_counts[:n].cpu().numpy()
    ov = d_ov.cpu().numpy()
    pairs = int(sum(int(counts[b]) * int(gt.counts[b]) for b in range(n)))
    nonzero = int(sum(int((ov[b, :counts[b], :gt.counts[b]] > 0).sum()) for b in range(n)))
    packed_pred = int(eng.packed_layout()[1])
    e2e = {}
    for name, thr in [("1", (0.5,)), ("10", thr10)]:
        t0 = time.perf_counter()
        reps = max(2, iters // 8)
        for _ in range(reps):
            res = api_utils.unmold_compute_ap_batch(items, gts, thr)
        e2e[name] = (time.perf_counter() - t0) / reps * 1e3
    matches = int(sum((r["pred_match"][0] > -1).sum() for r in res))
    rle = rle_gt_record(eng, gts, base_rle, base_n, items, thr10, iters)
    rec = {"workload":"configs[1] 32 x 1024x1024 x 100 predictions vs 100 jittered gt -> mask IoU, "
                       "matches, AP", "pairs": pairs, "pairs_with_overlap": nonzero,
           "matches_at_0.5": matches,
           "pred_packed_MB": round(packed_pred / 1e6, 1),
           "gt_packed_MB": round(int(gt.planes.d_packed.numel()) / 1e6, 1),
           "extents_kernel_ms": round(ext_ms, 4), "overlaps_ms_incl_pred_extents": round(ov_ms, 4),
           "matches_kernel_ms_1_threshold": round(m1_ms, 4),
           "matches_kernel_ms_10_thresholds": round(m10_ms, 4),
           "unmold_compute_ap_batch_ms_1_threshold": round(e2e["1"], 1),
           "unmold_compute_ap_batch_ms_10_thresholds": round(e2e["10"], 1),
           "note": "end to end: H2D of the inputs and of the bool gt masks (105 MB per image), "
                   "unmold, pack, scoring, downloads and the host AP tail", **rle, **card()}
    if cpu:
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
        import eval_oracle
        masks = api_utils.unmold_detections_batch(items[:1])[0][3]
        t0 = time.perf_counter()
        eval_oracle.compute_overlaps_masks(masks, gts[0][2])
        rec["cpu_oracle_compute_overlaps_masks_ms_per_image"] = round((time.perf_counter() - t0) * 1e3, 1)
    print(json.dumps(rec), flush=True)
    del eng, d_det, d_msk, gt, d_ov
    torch.cuda.empty_cache()


def cocoeval_case(iters, n_batches=4):
    """COCO mask AP over a stream of configs[1]-shaped batches: 32 x 1024x1024, 100 predictions
    against the 100 instances of the same image jittered, about 10 % of them crowd regions
    (synth.jitter_coco_ground_truth), default COCOeval params.  The three kernels alone on one
    batch, add_batch end to end per batch (input upload, unmold, packed expand, ground-truth
    decode, the kernels and the download), accumulate() over the whole stream, and the restated
    pycocotools evaluate (computeIoU + evaluateImg, tests/cocoeval_oracle.py) per image on the
    host."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate
    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import (coco_device_params,
                                                                         coco_evaluate_batch)

    batch, base_n = 32, 4
    base = synth.make_batch(11, base_n, (1024, 1024), 100)
    rng = np.random.default_rng(12)
    jit = [synth.jitter_coco_ground_truth(im, rng, crowd_frac=0.1, max_shift=12) for im in base]
    jit_items = [(j.detections, j.mrcnn_mask, j.original_image_shape, j.image_shape, j.window)
                 for j, _, _ in jit]
    gt_rle = api_utils.unmold_detections_rle_batch(jit_items, compressed=True)
    base_anns = [[{"category_id": int(c), "iscrowd": int(cr), "area": float(a), "segmentation": r}
                  for c, cr, a, r in zip(g[1], crowd, area, g[3])]
                 for g, (_, crowd, area) in zip(gt_rle, jit)]
    items = [(im.detections, im.mrcnn_mask, im.original_image_shape, im.image_shape, im.window)
             for im in (base[i % base_n] for i in range(batch))]
    anns = [base_anns[i % base_n] for i in range(batch)]
    ev = evaluate.COCOevalSegm()
    per_batch = []
    for k in range(n_batches):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev.add_batch(items, list(range(k * batch, (k + 1) * batch)), anns)
        per_batch.append((time.perf_counter() - t0) * 1e3)
    t0 = time.perf_counter()
    ev.accumulate()
    acc_ms = (time.perf_counter() - t0) * 1e3
    with open(os.devnull, "w") as null:
        stdout, sys.stdout = sys.stdout, null
        try:
            ev.summarize()
        finally:
            sys.stdout = stdout
    n_dets = int(sum(d[0].size for d in ev._dets))

    # the kernels alone on one planned batch
    eng = UnmoldEngine(batch, 100, (28, 28), 81)
    eng.plan([make_geom(*it[2:]) for it in items], canvas=False)
    d_det = torch.from_numpy(np.stack([it[0] for it in items])).cuda()
    d_msk = torch.from_numpy(np.stack([it[1] for it in items])).cuda()
    eng.enqueue_packed(d_det, d_msk)
    gt = eng.ground_truth_rle([np.array([a["category_id"] for a in x], np.int32) for x in anns],
                              [[a["segmentation"] for a in x] for x in anns])
    crowd = np.zeros((batch, gt.R), np.uint8)
    area = np.zeros((batch, gt.R))
    for b, x in enumerate(anns):
        crowd[b, :len(x)] = [a["iscrowd"] for a in x]
        area[b, :len(x)] = [a["area"] for a in x]
    pred = eng.predictions(gt)
    res = coco_evaluate_batch(eng.lib, pred.planes, pred.class_ids, pred.scores, gt, crowd, area,
                              np.arange(81, dtype=np.int32), ev.params)
    thr, rngs, max_det = coco_device_params(ev.params)
    n, R1, R2, T, A = batch, eng.R, gt.R, len(thr), len(rngs) // 2
    dev = eng.device
    d_map = torch.arange(81, dtype=torch.int32, device=dev)
    d_cat = torch.empty((n, R1), dtype=torch.int32, device=dev)
    d_rank, d_walk = torch.empty_like(d_cat), torch.empty_like(d_cat)
    d_keep = torch.empty((n, R1), dtype=torch.uint8, device=dev)
    d_crowd = torch.from_numpy(crowd).to(dev)
    d_area = torch.from_numpy(area).to(dev)
    d_pa = eng._eval_bufs["areas"]
    d_match = torch.empty((A, T, n, R1), dtype=torch.int32, device=dev)
    d_ign = torch.empty((A, T, n, R1), dtype=torch.uint8, device=dev)
    d_iou = res["d_iou"]
    st = N.stream_ptr(None)
    ranks = lambda: N.check(eng.lib.mrx_coco_ranks(  # noqa: E731
        eng.d_class_ids, eng.d_scores, N.MRX_F32, eng.d_counts, d_map, 81, max_det,
        d_cat, d_rank, d_keep, d_walk, n, R1, st), "mrx_coco_ranks")
    ious = lambda: N.check(eng.lib.mrx_coco_ious(  # noqa: E731
        eng.d_packed, eng.d_packed_off, eng.d_counts, d_pa,
        eng._eval_bufs["extents"], d_cat, d_keep, R1, gt.planes.d_packed,
        gt.planes.d_packed_off, gt.d_counts, gt.planes.d_areas, gt.planes.d_extents,
        gt.d_class_ids, d_crowd, R2, gt.d_geom, d_iou, n, st), "mrx_coco_ious")
    match = lambda: N.check(eng.lib.mrx_coco_match(  # noqa: E731
        d_iou, eng.d_counts, d_cat, d_keep, d_walk, d_pa, gt.d_counts,
        gt.d_class_ids, d_crowd, d_area, N.double_array(thr), T, N.double_array(rngs), A,
        d_match, d_ign, n, R1, R2, st), "mrx_coco_match")
    ranks()
    rank_ms, _ = time_ms(ranks, iters)
    iou_ms, _ = time_ms(ious, iters)
    match_ms, _ = time_ms(match, iters)

    # the restated pycocotools evaluate on the host, one image
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import cocoeval_oracle as co
    _, cls, scores, masks = api_utils.unmold_detections_batch(items[:1])[0]
    gts = [{"image_id": 0, "category_id": a["category_id"], "mask": gm, "iscrowd": a["iscrowd"],
            "area": a["area"]}
           for a, gm in zip(anns[0], np.moveaxis(api_utils.unmold_detections_batch(
               jit_items[:1])[0][3], 2, 0))]
    dts = [{"image_id": 0, "category_id": int(c), "mask": masks[:, :, i], "score": float(s)}
           for i, (c, s) in enumerate(zip(cls, scores))]
    oracle = co.COCOevalOracle(gts, dts)
    t0 = time.perf_counter()
    oracle.evaluate()
    host_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({
        "workload": f"COCOeval segm: {n_batches} batches of configs[1] 32 x 1024x1024, "
                    "100 predictions vs 100 jittered gt (~10 % crowd), default params",
        "detections_recorded": n_dets, "gt_crowd": int(sum(int(c.sum()) for _, c, _ in jit)) * (batch // base_n),
        "stats_0_AP": round(float(ev.stats[0]), 4),
        "ranks_kernel_ms": round(rank_ms, 4), "ious_kernel_ms": round(iou_ms, 4),
        "match_kernel_ms_40_area_thresholds": round(match_ms, 4),
        "add_batch_ms_per_batch": [round(t, 1) for t in per_batch],
        "accumulate_ms_whole_stream": round(acc_ms, 1),
        "host_oracle_evaluate_ms_per_image": round(host_ms, 1),
        "note": "add_batch: H2D of the configs[1] inputs (28x28x81 float32 tiles), unmold, packed "
                "expand, gt decode from compressed strings, the three kernels, one download",
        **card()}), flush=True)
    del eng, d_det, d_msk, gt, res, d_iou
    torch.cuda.empty_cache()


def coco_eval_inputs():
    """(batch, items, anns): the configs[1] batch of bboxeval_case and boundaryeval_case, 32 x
    1024x1024, 100 predictions against 100 jittered instances (~10 % crowd), annotated with
    compressed-RLE segmentations, areas and boxes (the jittered masks' extents with sub-pixel
    jitter, rounded to 2 decimals)."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils

    batch, base_n = 32, 4
    base = synth.make_batch(11, base_n, (1024, 1024), 100)
    rng = np.random.default_rng(12)
    jit = [synth.jitter_coco_ground_truth(im, rng, crowd_frac=0.1, max_shift=12) for im in base]
    jit_items = [(j.detections, j.mrcnn_mask, j.original_image_shape, j.image_shape, j.window)
                 for j, _, _ in jit]
    gt_rle = api_utils.unmold_detections_rle_batch(jit_items, compressed=True)
    base_anns = []
    for g, (_, crowd, area) in zip(gt_rle, jit):
        y1, x1, y2, x2 = g[0].astype(np.float64).T
        xywh = np.round(np.stack([x1, y1, x2 - x1, y2 - y1], 1)
                        + rng.uniform(-0.5, 0.5, (len(x1), 4)), 2)
        base_anns.append([{"category_id": int(c), "iscrowd": int(cr), "area": float(a),
                           "bbox": [float(v) for v in bb], "segmentation": r}
                          for c, cr, a, bb, r in zip(g[1], crowd, area, xywh, g[3])])
    items = [(im.detections, im.mrcnn_mask, im.original_image_shape, im.image_shape, im.window)
             for im in (base[i % base_n] for i in range(batch))]
    anns = [base_anns[i % base_n] for i in range(batch)]
    return batch, items, anns


def bboxeval_case(iters, n_batches=4):
    """COCO box AP over the batches of cocoeval_case (configs[1]: 32 x 1024x1024, 100 predictions
    against 100 jittered instances, ~10 % crowd), the ground-truth boxes the jittered masks'
    extents with sub-pixel jitter, rounded to 2 decimals.  The three kernels alone on one batch
    (ranks, box IoUs, match with float64 areas), COCOevalBbox.add_batch end to end per batch
    (input upload, unmold prepare, the kernels, the download; no mask), segm + bbox from one
    unmold (unmold_coco_eval_batch with both evaluators) against two separate add_batch calls, and
    the restated pycocotools bbox evaluate (tests/bbox_cocoeval_oracle.py) per image on the host."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate
    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import (coco_box_evaluate_batch,
                                                                         coco_device_params)

    batch, items, anns = coco_eval_inputs()

    def stream(make, add):
        evs, ts = make(), []
        for k in range(n_batches):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            add(evs, list(range(k * batch, (k + 1) * batch)))
            ts.append((time.perf_counter() - t0) * 1e3)
        return evs, ts

    bbox_only = lambda evs, ids: evs[0].add_batch(items, ids, anns)  # noqa: E731
    (ev,), per_batch = stream(lambda: [evaluate.COCOevalBbox()], bbox_only)
    _, apart = stream(lambda: [evaluate.COCOevalSegm(), evaluate.COCOevalBbox()],
                      lambda evs, ids: [e.add_batch(items, ids, anns) for e in evs])
    both_evs, both = stream(lambda: [evaluate.COCOevalSegm(), evaluate.COCOevalBbox()],
                            lambda evs, ids: api_utils.unmold_coco_eval_batch(items, ids, anns, evs))
    with open(os.devnull, "w") as null:
        stdout, sys.stdout = sys.stdout, null
        try:
            for e in [ev] + both_evs:
                e.accumulate()
                e.summarize()
        finally:
            sys.stdout = stdout

    # the kernels alone on one planned batch, after the prepare step only
    eng = UnmoldEngine(batch, 100, (28, 28), 81)
    eng.plan([make_geom(*it[2:]) for it in items], canvas=False)
    d_det = torch.from_numpy(np.stack([it[0] for it in items])).cuda()
    d_msk = torch.from_numpy(np.stack([it[1] for it in items])).cuda()
    eng.enqueue(d_det, d_msk, expand=False)
    tables = ev._gt_tables(list(range(batch)), anns)
    g_counts, g_cat, g_boxes, g_crowd, g_area = ev._gt_arrays(tables)
    pred = eng.predictions()
    res = coco_box_evaluate_batch(eng.lib, pred.boxes, pred.counts, pred.class_ids, pred.scores,
                                  g_counts, g_cat, g_boxes, g_crowd, g_area,
                                  ev._class_map(81, None), ev.params)
    thr, rngs, max_det = coco_device_params(ev.params)
    n, R1, R2, T, A = batch, eng.R, g_cat.shape[1], len(thr), len(rngs) // 2
    dev = eng.device
    d_map = torch.from_numpy(ev._class_map(81, None)).to(dev)
    d_cat = torch.empty((n, R1), dtype=torch.int32, device=dev)
    d_rank, d_walk = torch.empty_like(d_cat), torch.empty_like(d_cat)
    d_keep = torch.empty((n, R1), dtype=torch.uint8, device=dev)
    d_gcount, d_gcat = torch.from_numpy(g_counts).to(dev), torch.from_numpy(g_cat).to(dev)
    d_gbox, d_crowd = torch.from_numpy(g_boxes).to(dev), torch.from_numpy(g_crowd).to(dev)
    d_area = torch.from_numpy(g_area).to(dev)
    d_pa = torch.empty((n, R1), dtype=torch.float64, device=dev)
    d_match = torch.empty((A, T, n, R1), dtype=torch.int32, device=dev)
    d_ign = torch.empty((A, T, n, R1), dtype=torch.uint8, device=dev)
    d_iou = res["d_iou"]
    st = N.stream_ptr(None)
    ranks = lambda: N.check(eng.lib.mrx_coco_ranks(  # noqa: E731
        eng.d_class_ids, eng.d_scores, N.MRX_F32, eng.d_counts, d_map, 81, max_det,
        d_cat, d_rank, d_keep, d_walk, n, R1, st), "mrx_coco_ranks")
    ious = lambda: N.check(eng.lib.mrx_coco_box_ious(  # noqa: E731
        eng.d_boxes, N.MRX_BOX_YXYX_I32, eng.d_counts, d_cat, d_keep, R1, d_gbox,
        d_gcount, d_gcat, d_crowd, R2, d_pa, d_iou, n, st), "mrx_coco_box_ious")
    match = lambda: N.check(eng.lib.mrx_coco_match_f64area(  # noqa: E731
        d_iou, eng.d_counts, d_cat, d_keep, d_walk, d_pa, d_gcount,
        d_gcat, d_crowd, d_area, N.double_array(thr), T, N.double_array(rngs), A,
        d_match, d_ign, n, R1, R2, st), "mrx_coco_match_f64area")
    ranks()
    rank_ms, _ = time_ms(ranks, iters)
    iou_ms, _ = time_ms(ious, iters)
    match_ms, _ = time_ms(match, iters)
    counts = eng.d_counts[:n].cpu().numpy()
    pairs = int(sum(int(counts[b]) * int(g_counts[b]) for b in range(n)))

    # the restated pycocotools bbox evaluate on the host, one image
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import bbox_cocoeval_oracle as bo
    boxes, cls, scores, _ = api_utils.unmold_detections_packed_batch(items[:1])[0]
    gts = [{"image_id": 0, "category_id": a["category_id"], "bbox": a["bbox"],
            "iscrowd": a["iscrowd"], "area": a["area"]} for a in anns[0]]
    dts = [{"image_id": 0, "category_id": int(c), "score": float(s),
            "bbox": [int(b[1]), int(b[0]), int(b[3] - b[1]), int(b[2] - b[0])]}
           for b, c, s in zip(boxes, cls, scores)]
    oracle = bo.COCOevalBboxOracle(gts, dts)
    t0 = time.perf_counter()
    oracle.evaluate()
    host_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({
        "workload": f"COCOeval bbox: {n_batches} batches of configs[1] 32 x 1024x1024, "
                    "100 predictions vs 100 jittered gt boxes (~10 % crowd), default params",
        "pairs_per_batch": pairs, "bbox_stats_0_AP": round(float(ev.stats[0]), 4),
        "segm_stats_0_AP": round(float(both_evs[0].stats[0]), 4),
        "ranks_kernel_ms": round(rank_ms, 4), "box_ious_kernel_ms": round(iou_ms, 4),
        "match_kernel_ms_40_area_thresholds": round(match_ms, 4),
        "bbox_add_batch_ms_per_batch": [round(t, 1) for t in per_batch],
        "segm_plus_bbox_one_unmold_ms_per_batch": [round(t, 1) for t in both],
        "segm_plus_bbox_two_add_batch_ms_per_batch": [round(t, 1) for t in apart],
        "host_oracle_bbox_evaluate_ms_per_image": round(host_ms, 1),
        "note": "add_batch: H2D of the configs[1] inputs (28x28x81 float32 tiles), unmold prepare, "
                "the three kernels, one download; segm also expands packed planes and decodes "
                "the gt strings", **card()}), flush=True)
    del eng, d_det, d_msk, res, d_iou
    torch.cuda.empty_cache()


def boundaryeval_case(iters, n_batches=4):
    """Boundary AP (COCOeval "boundary", dilation_ratio 0.02: d = 29 at 1024x1024) over the batches
    of bboxeval_case.  The kernels alone on one batch: the boundaries of the predictions (inside
    their boxes) and of the ground truth (whole image), and the boundary IoUs;
    COCOevalBoundary.add_batch end to end per batch; segm + bbox + boundary from one unmold
    against three separate add_batch calls; and the restated boundary_iou_api evaluate
    (tests/boundary_cocoeval_oracle.py, cv2 erosion) per image on the host."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, evaluate
    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import (
        boundary_dilation, coco_boundary_evaluate_batch, coco_device_params)

    batch, items, anns = coco_eval_inputs()

    def stream(make, add):
        evs, ts = make(), []
        for k in range(n_batches):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            add(evs, list(range(k * batch, (k + 1) * batch)))
            ts.append((time.perf_counter() - t0) * 1e3)
        return evs, ts

    three = lambda: [evaluate.COCOevalSegm(), evaluate.COCOevalBbox(),  # noqa: E731
                     evaluate.COCOevalBoundary()]
    (ev,), per_batch = stream(lambda: [evaluate.COCOevalBoundary()],
                              lambda evs, ids: evs[0].add_batch(items, ids, anns))
    _, apart = stream(three, lambda evs, ids: [e.add_batch(items, ids, anns) for e in evs])
    together, both = stream(three, lambda evs, ids: api_utils.unmold_coco_eval_batch(items, ids,
                                                                                      anns, evs))
    with open(os.devnull, "w") as null:
        stdout, sys.stdout = sys.stdout, null
        try:
            for e in [ev] + together:
                e.accumulate()
                e.summarize()
        finally:
            sys.stdout = stdout

    # the kernels alone on one planned batch
    eng = UnmoldEngine(batch, 100, (28, 28), 81)
    eng.plan([make_geom(*it[2:]) for it in items], canvas=False)
    d_det = torch.from_numpy(np.stack([it[0] for it in items])).cuda()
    d_msk = torch.from_numpy(np.stack([it[1] for it in items])).cuda()
    eng.enqueue_packed(d_det, d_msk)
    gt = eng.ground_truth_rle([np.array([a["category_id"] for a in x], np.int32) for x in anns],
                              [[a["segmentation"] for a in x] for x in anns])
    crowd = np.zeros((batch, gt.R), np.uint8)
    area = np.zeros((batch, gt.R))
    for b, x in enumerate(anns):
        crowd[b, :len(x)] = [a["iscrowd"] for a in x]
        area[b, :len(x)] = [a["area"] for a in x]
    bufs = eng._eval_bufs
    pred = eng.predictions(gt)
    res = coco_boundary_evaluate_batch(eng.lib, pred.planes, pred.boxes, pred.class_ids,
                                       pred.scores, gt, crowd, area, np.arange(81, dtype=np.int32),
                                       ev.params, bufs=bufs)
    thr, rngs, max_det = coco_device_params(ev.params)
    n, R1, R2 = batch, eng.R, gt.R
    dev = eng.device
    d_dil = torch.from_numpy(boundary_dilation(eng.layout.geom, 0.02)).to(dev)
    d_map = torch.arange(81, dtype=torch.int32, device=dev)
    d_cat = torch.empty((n, R1), dtype=torch.int32, device=dev)
    d_rank, d_walk = torch.empty_like(d_cat), torch.empty_like(d_cat)
    d_keep = torch.empty((n, R1), dtype=torch.uint8, device=dev)
    d_crowd = torch.from_numpy(crowd).to(dev)
    d_iou = res["d_iou"]
    st = N.stream_ptr(None)
    max_w = eng.layout.max_w
    N.check(eng.lib.mrx_coco_ranks(
        eng.d_class_ids, eng.d_scores, N.MRX_F32, eng.d_counts, d_map, 81, max_det,
        d_cat, d_rank, d_keep, d_walk, n, R1, st), "mrx_coco_ranks")
    pred_bnd = lambda: N.check(eng.lib.mrx_mask_boundary(  # noqa: E731
        eng.d_packed, eng.d_packed_off, eng.d_counts, eng.d_geom, eng.d_boxes,
        d_dil, bufs["pred_boundary_packed"], n, R1, max_w, st), "mrx_mask_boundary")
    gt_bnd = lambda: N.check(eng.lib.mrx_mask_boundary(  # noqa: E731
        gt.planes.d_packed, gt.planes.d_packed_off, gt.d_counts, gt.d_geom,
        gt.d_regions, d_dil, bufs["gt_boundary_packed"], n, R2, max_w, st),
        "mrx_mask_boundary")
    ious = lambda: N.check(eng.lib.mrx_coco_boundary_ious(  # noqa: E731
        eng.d_packed, eng.d_packed_off, eng.d_counts, bufs["areas"],
        bufs["extents"], bufs["pred_boundary_packed"], bufs["pred_boundary_areas"],
        d_cat, d_keep, R1, gt.planes.d_packed, gt.planes.d_packed_off,
        gt.d_counts, gt.planes.d_areas, gt.planes.d_extents,
        bufs["gt_boundary_packed"], bufs["gt_boundary_areas"], gt.d_class_ids,
        d_crowd, R2, gt.d_geom, d_iou, n, st), "mrx_coco_boundary_ious")
    pred_ms, _ = time_ms(pred_bnd, iters)
    gt_ms, _ = time_ms(gt_bnd, iters)
    iou_ms, _ = time_ms(ious, iters)
    gt_bytes = int(sum(int(gt.counts[b]) * int(gt.geom[b, 0]) * ((int(gt.geom[b, 1]) + 7) // 8)
                       for b in range(n)))

    # the restated boundary_iou_api evaluate on the host, one image
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import boundary_cocoeval_oracle as bo
    _, cls, scores, masks = api_utils.unmold_detections_batch(items[:1])[0]
    H, W = int(gt.geom[0, 0]), int(gt.geom[0, 1])
    wb = (W + 7) // 8
    host = gt.planes.d_packed[:int(gt.counts[0]) * H * wb].cpu().numpy().reshape(-1, H, wb)
    gt_masks = np.unpackbits(host, axis=2)[:, :, :W].astype(bool)
    gts = [{"image_id": 0, "category_id": a["category_id"], "mask": gm, "iscrowd": a["iscrowd"],
            "area": a["area"]} for a, gm in zip(anns[0], gt_masks)]
    dts = [{"image_id": 0, "category_id": int(c), "mask": masks[:, :, i], "score": float(s)}
           for i, (c, s) in enumerate(zip(cls, scores))]
    oracle = bo.COCOevalBoundaryOracle(gts, dts)
    t0 = time.perf_counter()
    oracle.evaluate()
    host_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({
        "workload": f"COCOeval boundary: {n_batches} batches of configs[1] 32 x 1024x1024, "
                    "100 predictions vs 100 jittered gt (~10 % crowd), default params, "
                    "dilation_ratio 0.02 (d = 29)",
        "boundary_stats_0_AP": round(float(ev.stats[0]), 4),
        "segm_stats_0_AP": round(float(together[0].stats[0]), 4),
        "pred_boundary_kernel_ms": round(pred_ms, 4),
        "gt_boundary_kernel_ms": round(gt_ms, 4),
        "gt_planes_MB": round(gt_bytes / 1e6, 1),
        "gt_boundary_read_plus_write_GBps": round(2 * gt_bytes / gt_ms / 1e6, 1),
        "boundary_ious_kernel_ms": round(iou_ms, 4),
        "boundary_add_batch_ms_per_batch": [round(t, 1) for t in per_batch],
        "segm_bbox_boundary_one_unmold_ms_per_batch": [round(t, 1) for t in both],
        "segm_bbox_boundary_three_add_batch_ms_per_batch": [round(t, 1) for t in apart],
        "host_oracle_boundary_evaluate_ms_per_image": round(host_ms, 1),
        "note": "add_batch: H2D of the configs[1] inputs, unmold, packed expand, gt decode from "
                "compressed strings, both boundary launches and their extents, ranks, boundary "
                "IoUs, match, one download", **card()}), flush=True)
    del eng, d_det, d_msk, gt, res, d_iou
    torch.cuda.empty_cache()


def rle_gt_record(eng, gts, base_rle, base_n, items, thr10, iters):
    """The ground truth of eval_case as COCO compressed strings: mrx_rle_parse, mrx_rle_decode
    and the whole-image mrx_mask_extents alone on the uploaded strings, and
    unmold_compute_ap_batch end to end with them in place of the bool masks."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils
    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import BatchLayout, pack_rle

    n, lib = len(gts), eng.lib
    rles = [base_rle[b % base_n] for b in range(n)]
    cls = [g[1] for g in gts]
    geom = eng.layout.geom
    pk = pack_rle(geom, cls, rles)
    R = pk["R"]
    layout = BatchLayout(geom, R, limits=False)
    dev = eng.device
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    d_str, d_str_off, d_run_off = up(pk["strings"]), up(pk["str_off"]), up(pk["run_off"])
    d_counts, d_geom = up(pk["counts"]), up(geom)
    d_run_count = up(pk["run_count"])
    d_status = torch.zeros((n * R,), dtype=torch.int32, device=dev)
    d_runs = torch.empty((pk["strings"].size,), dtype=torch.int32, device=dev)
    d_ends = torch.empty((pk["strings"].size,), dtype=torch.int64, device=dev)
    d_off = up(layout.packed_off[:-1])
    d_packed = torch.empty((int(layout.packed_off[-1]),), dtype=torch.uint8, device=dev)
    regions = np.zeros((n, R, 4), np.int32)
    regions[:, :, 2:] = geom[:, None, :2]
    d_regions = up(regions)
    d_areas = torch.empty((n, R), dtype=torch.int64, device=dev)
    d_ext = torch.empty((n, R, 4), dtype=torch.int32, device=dev)
    st = N.stream_ptr(None)

    def parse():
        N.check(lib.mrx_rle_parse(d_str, d_str_off, d_counts, d_runs, d_run_count,
                                  d_status, n, R, st), "mrx_rle_parse")

    def decode():
        N.check(lib.mrx_rle_decode(d_runs, d_run_off, d_run_count, d_ends, d_status,
                                   d_counts, d_geom, d_off, d_packed, n, R,
                                   layout.max_h, layout.max_w, st), "mrx_rle_decode")

    def extents():
        N.check(lib.mrx_mask_extents(d_packed, d_off, d_counts, d_geom, d_regions,
                                     d_areas, d_ext, n, R, st), "mrx_mask_extents")

    parse_ms, _ = time_ms(parse, iters)
    decode_ms, _ = time_ms(decode, iters)
    ext_ms, _ = time_ms(extents, iters)
    assert not d_status.any().item(), "the benchmark's strings must decode cleanly"
    rle_gts = [(g[0], g[1], r) for g, r in zip(gts, rles)]
    e2e = {}
    for name, thr in [("1", (0.5,)), ("10", thr10)]:
        reps = max(2, iters // 8)
        api_utils.unmold_compute_ap_batch(items, rle_gts, thr)
        t0 = time.perf_counter()
        for _ in range(reps):
            res = api_utils.unmold_compute_ap_batch(items, rle_gts, thr)
        e2e[name] = (time.perf_counter() - t0) / reps * 1e3
    want = api_utils.unmold_compute_ap_batch(items, gts, thr10)
    same = all(np.array_equal(a["pred_match"], b["pred_match"]) and
               np.array_equal(a["gt_match"], b["gt_match"]) for a, b in zip(res, want))
    packed = int(sum(layout.packed_span(b, pk["counts"][b])[1] - layout.packed_span(b, 0)[0]
                     for b in range(n)))
    return {"rle_gt_string_MB": round(pk["strings"].size / 1e6, 2),
            "rle_gt_instances": int(pk["counts"].sum()),
            "rle_parse_kernel_ms": round(parse_ms, 4),
            "rle_decode_kernels_ms": round(decode_ms, 4),
            "rle_decode_packed_write_GBps": round(packed / decode_ms / 1e6, 1),
            "rle_gt_extents_kernel_ms": round(ext_ms, 4),
            "unmold_compute_ap_batch_ms_1_threshold_rle_gt": round(e2e["1"], 1),
            "unmold_compute_ap_batch_ms_10_thresholds_rle_gt": round(e2e["10"], 1),
            "rle_gt_results_equal_bool_gt": bool(same)}


def _coco_like_polygons(rng, H, W, n):
    """n COCO-style polygon annotations: 1-3 parts of 10-60 vertices, star-shaped around a
    random centre (some reaching past the image)."""
    out = []
    for _ in range(n):
        parts = []
        for _ in range(int(rng.integers(1, 4))):
            v = int(rng.integers(10, 61))
            t = np.sort(rng.uniform(0, 2 * np.pi, v))
            r = rng.uniform(5, 0.3 * min(H, W)) * rng.uniform(0.6, 1.0, v)
            cx, cy = rng.uniform(0, W), rng.uniform(0, H)
            parts.append(np.round(np.stack([cx + r * np.cos(t), cy + r * np.sin(t)], 1), 2)
                         .ravel().tolist())
        out.append(parts)
    return out


def _contour_polygons(contours):
    """A display_instances contour list as a COCO polygon list: parts of >= 3 vertices (an
    instance with none gets one degenerate part, an empty mask)."""
    parts = [c.ravel().tolist() for c in contours if len(c) >= 3]
    return parts or [[0.0, 0.0, 0.0, 0.0, 0.0, 0.0]]


def polygons_case(iters):
    """COCO polygon ground truth rasterised on the device (mrx_poly_decode).  COCO-like: 32 x
    640x480 images of 5-20 annotations (1-3 parts of 10-60 vertices).  configs[1]: the jittered
    ground truth of eval_case as the contour polygons of unmold_detections_contours_batch.  The
    kernels alone, MaskBatch.from_coco end to end, unmold_compute_ap_batch with the polygons
    against the same batch with RLE strings, and the polygon oracle's host time per image."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils
    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import MaskBatch, pack_polygons

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import polygon_oracle

    lib, dev = N.load(), torch.device("cuda", 0)
    rng = np.random.default_rng(12)
    rec = {"workload": "COCO polygon ground truth -> packed planes (pycocotools annToRLE + decode)"}

    def kernels_ms(geoms, cls, segms):
        pp = pack_polygons(geoms, cls, segms)
        gt = MaskBatch.from_coco(lib, dev, geoms, cls, segms)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        t = [up(pp[k]) for k in ("vert", "part_vert", "part_inst", "part_col", "part_tog",
                                 "inst_part")]
        d_tog = torch.empty((int(pp["part_tog"][-1]),), dtype=torch.int32, device=dev)
        d_cs = torch.empty((int(pp["part_col"][-1]),), dtype=torch.int64, device=dev)
        d_cy = torch.empty((int(pp["part_col"][-1]),), dtype=torch.uint8, device=dev)
        g = np.asarray(geoms)
        pl = gt.planes

        def run():
            N.check(lib.mrx_poly_decode(t[0], t[1], t[2], t[3], t[4], pp["P"],
                                        t[5], d_tog, d_cs, d_cy, pl.d_counts,
                                        gt.d_geom, pl.d_packed_off, pl.d_packed, len(g),
                                        gt.R, int(g[:, 0].max()), int(g[:, 1].max()),
                                        N.stream_ptr(None)), "mrx_poly_decode")
        ms, _ = time_ms(run, iters)

        def e2e():
            MaskBatch.from_coco(lib, dev, geoms, cls, segms)
        e2e()
        t0 = time.perf_counter()
        reps = max(3, iters // 4)
        for _ in range(reps):
            e2e()
        return pp, ms, (time.perf_counter() - t0) / reps * 1e3

    # 1. COCO-like
    H, W = 480, 640
    segms = [_coco_like_polygons(rng, H, W, int(rng.integers(5, 21))) for _ in range(32)]
    cls = [np.ones(len(s), np.int32) for s in segms]
    geoms = [[H, W, H, W, 0, 0, H, W]] * 32
    pp, k_ms, e_ms = kernels_ms(geoms, cls, segms)
    t0 = time.perf_counter()
    for s in segms[0]:
        polygon_oracle.ann_to_rle(s, H, W)
    rec.update({"coco_like_images": 32, "coco_like_instances": int(pp["counts"].sum()),
                "coco_like_parts": pp["P"], "coco_like_vertices": int(pp["vert"].shape[0]),
                "coco_like_poly_decode_kernels_ms": round(k_ms, 4),
                "coco_like_from_coco_ms": round(e_ms, 2),
                "oracle_host_ms_per_image": round((time.perf_counter() - t0) * 1e3, 1)})

    # 2. configs[1] ground truth as contour polygons
    batch, base_n = 32, 4
    base = synth.make_batch(7, base_n, (1024, 1024), 100)
    jrng = np.random.default_rng(8)
    jittered = [(j.detections, j.mrcnn_mask, j.original_image_shape, j.image_shape, j.window)
                for j in (synth.jitter_ground_truth(im, jrng, 12, 0.1) for im in base)]
    cont = api_utils.unmold_detections_contours_batch(jittered)
    polys = [[_contour_polygons(c) for c in r[3]] for r in cont]
    items = [(im.detections, im.mrcnn_mask, im.original_image_shape, im.image_shape, im.window)
             for im in (base[i % base_n] for i in range(batch))]
    gcls = [cont[i % base_n][1] for i in range(batch)]
    gp = [(None, gcls[i], polys[i % base_n]) for i in range(batch)]
    # the RLE of the same polygons, so that both routes score identical masks
    rle_of = [[{"size": [1024, 1024], "counts": polygon_oracle.ann_to_rle(s, 1024, 1024)}
               for s in polys[b]] for b in range(base_n)]
    gr = [(None, gcls[i], rle_of[i % base_n]) for i in range(batch)]
    geoms = [[1024, 1024, 1024, 1024, 0, 0, 1024, 1024]] * batch
    pp, k_ms, e_ms = kernels_ms(geoms, gcls, [polys[i % base_n] for i in range(batch)])
    e2e = {}
    for name, g in (("polygon_gt", gp), ("rle_gt", gr)):
        api_utils.unmold_compute_ap_batch(items, g, (0.5,))
        reps = max(2, iters // 8)
        t0 = time.perf_counter()
        for _ in range(reps):
            res = api_utils.unmold_compute_ap_batch(items, g, (0.5,))
        e2e[name] = ((time.perf_counter() - t0) / reps * 1e3, res)
    same = all(np.array_equal(a["gt_match"], b["gt_match"]) and
               np.array_equal(a["pred_match"], b["pred_match"])
               for a, b in zip(e2e["polygon_gt"][1], e2e["rle_gt"][1]))
    rec.update({"configs1_instances": int(pp["counts"].sum()), "configs1_parts": pp["P"],
                "configs1_vertices": int(pp["vert"].shape[0]),
                "configs1_poly_decode_kernels_ms": round(k_ms, 4),
                "configs1_from_coco_ms": round(e_ms, 2),
                "unmold_compute_ap_batch_ms_1_threshold_polygon_gt": round(e2e["polygon_gt"][0], 1),
                "unmold_compute_ap_batch_ms_1_threshold_rle_list_gt": round(e2e["rle_gt"][0], 1),
                "polygon_gt_results_equal_rle_gt": bool(same), **card()})
    print(json.dumps(rec), flush=True)
    torch.cuda.empty_cache()


def _lvis_dataset(rng, n_img, K=1203):
    """LVIS-like category dicts (v1's split: 337 rare, 461 common, 405 frequent) and image dicts
    of n_img 1024x1024 images, each with ~20 negative and ~2 not-exhaustive categories."""
    freq = np.array(["r"] * 337 + ["c"] * 461 + ["f"] * 405)[rng.permutation(K)]
    cats = [{"id": k + 1, "frequency": str(freq[k])} for k in range(K)]
    images = [{"id": i, "height": 1024, "width": 1024,
               "neg_category_ids": [int(c) for c in rng.choice(K, 20, replace=False) + 1],
               "not_exhaustive_category_ids": [int(c) for c in rng.choice(K, 2, replace=False) + 1]}
              for i in range(n_img)]
    return cats, images


def lvis_case(iters, n_batches=4, batch=32, R=300):
    """LVIS mask AP (LVISEvalSegm) on 32 x 1024x1024 images with 300 predictions each and
    jittered polygon ground truth (a 4-vertex polygon around every third predicted box, 100 per
    image, 15 % of them with another category), 1 203 categories, and neg / not-exhaustive lists.
    The three device kernels alone on one planned batch (mrx_lvis_ranks over K = 1 203 with the
    predictions' categories spread over all 1 203, mrx_coco_ious, mrx_coco_match),
    LVISEvalSegm.add_batch end to end per batch, and the host accumulate() + summarize() on
    synthetic records at LVIS-val scale (20 000 images x 300 detections, 1 203 categories)."""
    from matterport_maskrcnn_with_tensorflow_serving_b200 import evaluate
    from matterport_maskrcnn_with_tensorflow_serving_b200.engine import lvis_device_params

    rng = np.random.default_rng(11)
    K = 1203
    ims = [synth.make_image(rng, (1024, 1024), R, num_classes=81, max_instances=R)
           for _ in range(batch)]
    items = [(im.detections.astype(np.float32), im.mrcnn_mask.astype(np.float32),
              im.original_image_shape, im.image_shape, im.window) for im in ims]
    cmap81 = [0] + [int(c) for c in rng.choice(K, 80, replace=False) + 1]   # class -> category
    lvis_cls = rng.integers(1, K + 1, size=(batch, R)).astype(np.int32)      # for the kernels
    cats, images = _lvis_dataset(rng, n_batches * batch)
    segs, cls81, cls_all = [], [], []
    for b, im in enumerate(ims):
        det = im.detections
        s, c1, c2 = [], [], []
        for k in range(0, im.n_valid, 3):
            y1, x1, y2, x2 = (det[k, :4] * 1024 + rng.integers(-6, 7, 4)).tolist()
            s.append([[x1, y1, x2, y1 + 3, x2 - 4, y2, x1 + 2, y2 - 2]])
            flip = rng.random() < 0.15
            c1.append(int(rng.integers(1, 81)) if flip else int(det[k, 4]))
            c2.append(int(rng.integers(1, K + 1)) if flip else int(lvis_cls[b, k]))
        segs.append(s)
        cls81.append(c1)
        cls_all.append(c2)
    anns = [[{"category_id": cmap81[c], "segmentation": sg, "area": 5000.0, "iscrowd": 0}
             for c, sg in zip(c1, s)] for c1, s in zip(cls81, segs)]

    per_batch, ev = [], evaluate.LVISEvalSegm(cats, images)
    for k in range(n_batches):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev.add_batch(items, list(range(k * batch, (k + 1) * batch)), anns, category_ids=cmap81)
        per_batch.append((time.perf_counter() - t0) * 1e3)
    ev.run()

    # the kernels alone on one planned batch, every category of the 1 203 in play
    eng = UnmoldEngine(batch, R, (28, 28), 81)
    eng.plan([make_geom(*it[2:]) for it in items], canvas=False)
    d_det = torch.from_numpy(np.stack([it[0] for it in items])).cuda()
    d_msk = torch.from_numpy(np.stack([it[1] for it in items])).cuda()
    eng.enqueue_packed(d_det, d_msk)
    gt_dense = [np.asarray(c, np.int32) - 1 for c in cls_all]
    gt = eng.ground_truth_coco(gt_dense, segs)
    pred = eng.predictions(gt).planes
    status = ev.status_table(list(range(batch)), gt_dense)
    thr, rngs, max_det = lvis_device_params(ev.params)
    n, R1, R2, T, A = batch, eng.R, gt.R, len(thr), len(rngs) // 2
    dev = eng.device
    d_cls = torch.from_numpy(lvis_cls).to(dev)
    d_map = torch.arange(-1, K, dtype=torch.int32, device=dev)      # category id -> dense
    d_status = torch.from_numpy(status).to(dev)
    d_cat = torch.empty((n, R1), dtype=torch.int32, device=dev)
    d_rank, d_walk = torch.empty_like(d_cat), torch.empty_like(d_cat)
    d_keep = torch.empty((n, R1), dtype=torch.uint8, device=dev)
    d_crowd = torch.zeros((n, R2), dtype=torch.uint8, device=dev)
    d_area = torch.full((n, R2), 5000.0, dtype=torch.float64, device=dev)
    d_match = torch.empty((A, T, n, R1), dtype=torch.int32, device=dev)
    d_ign = torch.empty((A, T, n, R1), dtype=torch.uint8, device=dev)
    d_iou = torch.empty((n, R1, R2), dtype=torch.float64, device=dev)
    st = N.stream_ptr(None)
    ranks = lambda: N.check(eng.lib.mrx_lvis_ranks(  # noqa: E731
        d_cls, eng.d_scores, N.MRX_F32, eng.d_counts, d_map, K + 1, d_status, K,
        max_det, d_cat, d_rank, d_keep, d_walk, n, R1, st), "mrx_lvis_ranks")
    ious = lambda: N.check(eng.lib.mrx_coco_ious(  # noqa: E731
        pred.d_packed, pred.d_packed_off, pred.d_counts, pred.d_areas,
        pred.d_extents, d_cat, d_keep, R1, gt.planes.d_packed,
        gt.planes.d_packed_off, gt.planes.d_counts, gt.planes.d_areas,
        gt.planes.d_extents, gt.d_class_ids, d_crowd, R2, gt.d_geom, d_iou, n,
        st), "mrx_coco_ious")
    match = lambda: N.check(eng.lib.mrx_coco_match(  # noqa: E731
        d_iou, eng.d_counts, d_cat, d_keep, d_walk, pred.d_areas,
        gt.planes.d_counts, gt.d_class_ids, d_crowd, d_area, N.double_array(thr), T,
        N.double_array(rngs), A, d_match, d_ign, n, R1, R2, st), "mrx_coco_match")
    ranks()
    rank_ms, _ = time_ms(ranks, iters)
    iou_ms, _ = time_ms(ious, iters)
    match_ms, _ = time_ms(match, iters)
    kept = int(d_keep.sum().item())
    cat_h, keep_h = d_cat.cpu().numpy(), d_keep.cpu().numpy().astype(bool)
    pairs = int(sum(np.sum(cat_h[b][keep_h[b]][:, None] == gt_dense[b][None, :])
                    for b in range(n)))
    del eng, d_det, d_msk, gt, pred, d_iou
    torch.cuda.empty_cache()

    # host accumulate + summarize at LVIS-val scale on synthetic records
    n_img, D, G, T, A = 20000, 300, 12, 10, 4
    host = evaluate.LVISEvalSegm(cats, _lvis_dataset(rng, n_img)[1])
    host._img_index = {i: i for i in range(n_img)}
    d_img = np.repeat(np.arange(n_img, dtype=np.int64), D)
    d_cat = rng.integers(0, K, size=n_img * D).astype(np.int32)
    d_score = np.round(rng.random(n_img * D), 3)
    order = np.lexsort((-d_score, d_cat, d_img))
    d_rank = np.empty(n_img * D, np.int32)
    first = np.r_[True, (d_img[order][1:] != d_img[order][:-1])
                  | (d_cat[order][1:] != d_cat[order][:-1])]
    run = np.cumsum(first) - 1
    start = np.flatnonzero(first)
    d_rank[order] = np.arange(n_img * D) - start[run]
    d_tp = rng.random((n_img * D, A, T)) < 0.3
    d_ig = rng.random((n_img * D, A, T)) < 0.1
    host._dets = [(d_img, d_cat, d_rank, d_score, d_tp, d_ig)]
    host._gts = [(np.repeat(np.arange(n_img, dtype=np.int64), G),
                  rng.integers(0, K, size=n_img * G).astype(np.int32),
                  rng.random((n_img * G, A)) < 0.8)]
    host._sync_params()
    t0 = time.perf_counter()
    host.accumulate()
    host.summarize()
    host_s = time.perf_counter() - t0
    print(json.dumps({
        "workload": f"LVISEval segm: {n_batches} batches of 32 x 1024x1024, 300 predictions vs "
                    "100 jittered polygon gt, 1 203 categories, neg / not-exhaustive lists",
        "kept_predictions_per_batch_kernels": kept, "pairs_per_batch_kernels": pairs,
        "lvis_ranks_kernel_ms": round(rank_ms, 4), "ious_kernel_ms": round(iou_ms, 4),
        "match_kernel_ms_40_area_thresholds": round(match_ms, 4),
        "add_batch_ms_per_batch": [round(t, 1) for t in per_batch],
        "AP": round(float(ev.results["AP"]), 4),
        "host_accumulate_summarize_s_20000_images_x_300": round(host_s, 2),
        "note": "add_batch: the model's 81 mask classes mapped onto 80 of the 1 203 categories "
                "(a 1 204-class mask head input would be 1.1 GB per image); H2D of the inputs, "
                "unmold prepare, packed expand, polygon rasterisation, the three kernels, one "
                "download", **card()}), flush=True)


def anchors_sweep(iters, cpu):
    import oracle
    gen = AnchorGenerator(MaskRCNNServingConfig)
    for s in [512, 640, 768, 896, 1000, 1024, 1280, 1536, 1792, 2000, 2048]:
        shape = (s, s, 3)
        n = gen.count(shape)
        out = torch.empty((n, 4), dtype=torch.float32, device="cuda")
        med, best = time_ms(lambda: gen.generate_device(shape, out=out), iters)
        rec = {"workload": "configs[4] get_anchors", "size": s, "anchors": int(n),
               "gpu_us_per_call": round(med * 1e3, 2), "gpu_Ganchors_per_s": round(n / med / 1e6, 2),
               "gpu_write_GBps": round(n * 16 / med / 1e6, 1)}
        if cpu:
            t0 = time.perf_counter()
            reps = 3
            for _ in range(reps):
                oracle.get_anchors(shape)
            cpu_ms = (time.perf_counter() - t0) / reps * 1e3
            rec["cpu_oracle_ms_per_call"] = round(cpu_ms, 3)
            rec["cpu_Manchors_per_s"] = round(n / cpu_ms / 1e3, 2)
        print(json.dumps(rec), flush=True)


def mold_cases(iters, cpu):
    import oracle
    rng = np.random.default_rng(2)
    m = Molder(MaskRCNNServingConfig)
    for hw in [(1024, 1024), (800, 1333), (2160, 3840)]:
        img = synth.synth_rgb_image(rng, *hw)
        d_img = torch.from_numpy(img).cuda()
        med, _ = time_ms(lambda: m.mold_device(d_img, np.float32), iters)
        rec = {"workload": "mold step (resize_image + mold_image, f32 out)", "hw": list(hw),
               "gpu_us_per_image": round(med * 1e3, 2),
               "algorithmic_GBps": round((3 * hw[0] * hw[1] + 12 * 1024 * 1024) / med / 1e6, 1)}
        if cpu:
            t0 = time.perf_counter()
            u8, *_ = oracle.resize_image(img, min_dim=800, max_dim=1024, min_scale=0, mode="square")
            oracle.mold_image(u8)
            rec["cpu_oracle_ms_per_image"] = round((time.perf_counter() - t0) * 1e3, 2)
        print(json.dumps(rec), flush=True)
    img = synth.synth_rgb_image(rng, 1080, 1920)
    d_img = torch.from_numpy(img).cuda()
    med, _ = time_ms(lambda: m.cv2_resize_device(d_img, (640, 640)), iters)
    print(json.dumps({"workload": "cv2.resize 1080x1920 -> 640x640 (u8, INTER_LINEAR)",
                      "gpu_us_per_image": round(med * 1e3, 2)}), flush=True)


def jpeg_case(iters):
    """JPEG request bytes decoded on the device (csrc/jpeg.cu) against cv2.imdecode on the host,
    each followed by preprocess_input_batch: 32 x 1024^2 and 16 x 2160x3840, quality 90, 4:2:0,
    no restart markers (cv2.imencode's defaults)."""
    import cv2
    from concurrent.futures import ThreadPoolExecutor

    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, jpeg, serve

    rng = np.random.default_rng(11)
    params = [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
              cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420]
    m = Molder(api_utils.get_config())
    for name, batch, hw in [("32 x 1024x1024", 32, (1024, 1024)),
                            ("configs[3] size: 16 x 2160x3840", 16, (2160, 3840))]:
        base = [synth.synth_rgb_image(rng, *hw) for _ in range(4)]
        blobs = [cv2.imencode(".jpg", base[b % 4][:, :, ::-1], params)[1].tobytes()
                 for b in range(batch)]
        mb = sum(len(b) for b in blobs) / 1e6
        # S sweep: Molder.decode_jpeg_batch, host parse and status read included
        sweep = {}
        for S in (256, 512, 1024, 2048, 4096):
            sweep[S], _ = time_ms(lambda: m.decode_jpeg_batch(blobs, S=S), iters)
        # kernel times, one profiled run of its own
        from torch.profiler import ProfilerActivity, profile
        m.decode_jpeg_batch(blobs)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                m.decode_jpeg_batch(blobs)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "jpeg_" in ev.key:
                short = ev.key.split("jpeg_")[1].split("_kernel")[0]
                kern[short] = round(ev.device_time_total / 1e3 / 5, 4)
        plan = jpeg.Plan(blobs)
        # sync rounds (largest over an image's CTAs) and the walk's re-decoded subsequences, per
        # image, from the counters the kernels leave after each image's subsequence arrays
        m.decode_jpeg_batch(blobs)
        work = m._jpeg_bufs["work"].cpu().numpy()
        tail = [int(plan.desc[b, jpeg.D_SUB_OFF] + 4 * plan.desc[b, jpeg.D_SUB_CAP])
                for b in range(batch)]
        rounds = [int(work[t + 1]) for t in tail]
        redone = [int(work[t + 2]) for t in tail]
        dec_ms, _ = time_ms(lambda: api_utils.decode_jpeg_batch(blobs), iters)
        pre_ms, _ = time_ms(lambda: serve.preprocess_input_batch(blobs), iters)

        def host(pool):
            dec = (lambda b: cv2.cvtColor(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR),
                                          cv2.COLOR_BGR2RGB))
            arrs = list(pool.map(dec, blobs)) if pool else [dec(b) for b in blobs]
            return serve.preprocess_input_batch(arrs)

        def host_clock(fn, n):
            fn()
            ts = []
            for _ in range(n):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            return float(np.median(ts))

        one_ms = host_clock(lambda: host(None), max(3, iters // 4))
        with ThreadPoolExecutor(os.cpu_count()) as pool:
            pool_ms = host_clock(lambda: host(pool), max(3, iters // 4))
        t_dec = time.perf_counter()
        cv2.imdecode(np.frombuffer(blobs[0], np.uint8), cv2.IMREAD_COLOR)
        imdecode_ms = (time.perf_counter() - t_dec) * 1e3
        print(json.dumps({
            "workload": f"JPEG decode {name} q90 4:2:0, no RST ({mb:.1f} MB of files)",
            "kernel_ms": kern, "subsequences_per_image_at_default_S": int(plan.max_subs),
            "default_S": jpeg.DEFAULT_S,
            "sync_rounds_per_image_min_median_max": [min(rounds), int(np.median(rounds)),
                                                     max(rounds)],
            "walk_redecoded_subsequences_per_image_min_median_max": [
                min(redone), int(np.median(redone)), max(redone)],
            "molder_decode_ms_by_S": {str(k): round(v, 3) for k, v in sweep.items()},
            "api_utils_decode_jpeg_batch_ms": round(dec_ms, 3),
            "preprocess_input_batch_bytes_ms": round(pre_ms, 3),
            "host_imdecode_one_thread_then_preprocess_ms": round(one_ms, 3),
            "host_imdecode_pool_then_preprocess_ms": round(pool_ms, 3),
            "host_threads": os.cpu_count(), "one_imdecode_ms": round(imdecode_ms, 3),
            **card()}), flush=True)


def jpeg_progressive_case(iters):
    """Progressive JPEG request bytes (cv2's IMWRITE_JPEG_PROGRESSIVE script) decoded on the device
    against cv2.imdecode on the host, each followed by preprocess_input_batch: 32 x 1024^2 and
    16 x 2160x3840, quality 90, 4:2:0, no restart markers.  Without restart markers every scan of an
    image is one serial unit, so the per-image chain of scans bounds the decode."""
    import cv2
    from concurrent.futures import ThreadPoolExecutor

    from torch.profiler import ProfilerActivity, profile

    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, jpeg, serve

    rng = np.random.default_rng(12)
    params = [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
              cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    m = Molder(api_utils.get_config())
    for name, batch, hw in [("32 x 1024x1024", 32, (1024, 1024)),
                            ("configs[3] size: 16 x 2160x3840", 16, (2160, 3840))]:
        base = [synth.synth_rgb_image(rng, *hw) for _ in range(4)]
        blobs = [cv2.imencode(".jpg", base[b % 4][:, :, ::-1], params)[1].tobytes()
                 for b in range(batch)]
        mb = sum(len(b) for b in blobs) / 1e6
        m.decode_jpeg_batch(blobs)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                m.decode_jpeg_batch(blobs)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "jpeg_" in ev.key:
                short = ev.key.split("jpeg_")[1].split("_kernel")[0]
                kern[short] = round(kern.get(short, 0) + ev.device_time_total / 1e3 / 5, 4)
        total = sum(kern.values())
        plan_ms = []
        for _ in range(max(3, iters // 4)):
            t0 = time.perf_counter()
            jpeg.plan_batch(blobs)
            plan_ms.append((time.perf_counter() - t0) * 1e3)
        dec_ms, _ = time_ms(lambda: api_utils.decode_jpeg_batch(blobs), iters)
        pre_ms, _ = time_ms(lambda: serve.preprocess_input_batch(blobs), iters)

        def host(pool):
            dec = (lambda b: cv2.cvtColor(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR),
                                          cv2.COLOR_BGR2RGB))
            arrs = list(pool.map(dec, blobs)) if pool else [dec(b) for b in blobs]
            return serve.preprocess_input_batch(arrs)

        def host_clock(fn, n):
            fn()
            ts = []
            for _ in range(n):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            return float(np.median(ts))

        one_ms = host_clock(lambda: host(None), max(3, iters // 4))
        with ThreadPoolExecutor(16) as pool:
            pool_ms = host_clock(lambda: host(pool), max(3, iters // 4))
        print(json.dumps({
            "workload": f"progressive JPEG decode {name} q90 4:2:0, no RST ({mb:.1f} MB of files)",
            "kernel_ms": kern, "kernel_ms_total": round(total, 3),
            "serial_decode_share": round(kern.get("prog_decode", 0) / total, 3) if total else None,
            "host_plan_ms": round(float(np.median(plan_ms)), 3),
            "api_utils_decode_jpeg_batch_ms": round(dec_ms, 3),
            "preprocess_input_batch_bytes_ms": round(pre_ms, 3),
            "host_imdecode_one_thread_then_preprocess_ms": round(one_ms, 3),
            "host_imdecode_16_threads_then_preprocess_ms": round(pool_ms, 3),
            "host_threads": os.cpu_count(), **card()}), flush=True)


def png_case(iters):
    """Overlay PNG files encoded on the device (csrc/png.cu) against cv2.imencode on the host:
    32 x 1024^2 and 16 x 2160x3840 overlays, and the tail of do_inference_batch that changed
    (unmold + overlay + PNG files written) before (overlays downloaded, cv2.imwrite) and after
    (encoded on the device, bytes written)."""
    import tempfile
    from concurrent.futures import ThreadPoolExecutor

    import cv2

    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, visualize

    from torch.profiler import ProfilerActivity, profile

    for name, batch, hw, n in [("32 x 1024x1024", 32, (1024, 1024), 100),
                               ("configs[3] size: 16 x 2160x3840", 16, (2160, 3840), 50)]:
        ims = synth.make_batch(5, 4, hw, n, num_classes=81)
        items = [(ims[b % 4].detections, ims[b % 4].mrcnn_mask, ims[b % 4].original_image_shape,
                  ims[b % 4].image_shape, ims[b % 4].window) for b in range(batch)]
        rng = np.random.default_rng(3)
        base = [synth.synth_rgb_image(rng, *hw) for _ in range(4)]
        images = [base[b % 4] for b in range(batch)]
        colors = visualize.random_colors(n)
        overlays = [o[3] for o in api_utils.unmold_overlay_batch(items[:4], images[:4], colors)]
        host = [overlays[b % 4] for b in range(batch)]
        dev = [torch.from_numpy(h).cuda() for h in host]
        files = api_utils.encode_png_batch(dev)
        mb = sum(len(f) for f in files) / 1e6
        api_utils.encode_png_batch(dev)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                api_utils.encode_png_batch(dev)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "png_" in ev.key:
                short = ev.key.split("png_")[1].split("_kernel")[0]
                kern[short] = round(kern.get(short, 0) + ev.device_time_total / 1e3 / 5, 4)
        enc_ms, _ = time_ms(lambda: api_utils.encode_png_batch(dev), iters)

        def host_clock(fn, k):
            fn()
            ts = []
            for _ in range(k):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            return float(np.median(ts))

        enc = lambda a: cv2.imencode(".png", a[:, :, ::-1])[1]     # noqa: E731
        k = max(3, iters // 4)
        one_ms = host_clock(lambda: [enc(a) for a in host], k)
        with ThreadPoolExecutor(16) as pool:
            pool_ms = host_clock(lambda: list(pool.map(enc, host)), k)
        with tempfile.TemporaryDirectory() as tmp:
            def before():
                outs = api_utils.unmold_overlay_batch(items, images, colors)
                for b, o in enumerate(outs):
                    cv2.imwrite(os.path.join(tmp, f"{b}.png"), o[3][:, :, ::-1])

            def after():
                outs = api_utils._unmold_overlay_file_batch(items, images, colors)
                for b, o in enumerate(outs):
                    with open(os.path.join(tmp, f"{b}.png"), "wb") as f:
                        f.write(o[3])

            before_ms = host_clock(before, k)
            after_ms = host_clock(after, k)
        print(json.dumps({
            "workload": f"PNG encode {name} overlays ({mb:.1f} MB of files)",
            "kernel_ms": kern, "kernel_ms_total": round(sum(kern.values()), 3),
            "api_utils_encode_png_batch_ms": round(enc_ms, 3),
            "host_imencode_one_thread_ms": round(one_ms, 3),
            "host_imencode_16_threads_ms": round(pool_ms, 3),
            "do_inference_batch_tail_before_ms": round(before_ms, 3),
            "do_inference_batch_tail_after_ms": round(after_ms, 3),
            "host_threads": os.cpu_count(), **card()}), flush=True)


def jpeg_encode_case(iters):
    """Overlay JPEG files encoded on the device (csrc/jpeg_encode.cu) at cv2's defaults against
    cv2.imencode('.jpg') on the host: 32 x 1024^2 and 16 x 2160x3840 overlays, their bytes
    against the device PNG of the same overlays, and the tail of do_inference_batch (unmold +
    overlay + files written) with image_format "jpeg" against "png"."""
    import tempfile
    from concurrent.futures import ThreadPoolExecutor

    import cv2

    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, visualize
    from matterport_maskrcnn_with_tensorflow_serving_b200 import jpeg_encode as je

    from torch.profiler import ProfilerActivity, profile

    for name, batch, hw, n in [("32 x 1024x1024", 32, (1024, 1024), 100),
                               ("configs[3] size: 16 x 2160x3840", 16, (2160, 3840), 50)]:
        ims = synth.make_batch(5, 4, hw, n, num_classes=81)
        items = [(ims[b % 4].detections, ims[b % 4].mrcnn_mask, ims[b % 4].original_image_shape,
                  ims[b % 4].image_shape, ims[b % 4].window) for b in range(batch)]
        rng = np.random.default_rng(3)
        base = [synth.synth_rgb_image(rng, *hw) for _ in range(4)]
        images = [base[b % 4] for b in range(batch)]
        colors = visualize.random_colors(n)
        overlays = [o[3] for o in api_utils.unmold_overlay_batch(items[:4], images[:4], colors)]
        host = [overlays[b % 4] for b in range(batch)]
        dev = [torch.from_numpy(h).cuda() for h in host]
        files = api_utils.encode_jpeg_batch(dev)
        enc = lambda a: cv2.imencode(".jpg", a[:, :, ::-1])[1]     # noqa: E731
        same = all(f == enc(h).tobytes() for f, h in zip(files[:4], host[:4]))
        jpeg_mb = sum(len(f) for f in files) / 1e6
        png_mb = sum(len(f) for f in api_utils.encode_png_batch(dev)) / 1e6
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                api_utils.encode_jpeg_batch(dev)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "jpeg_" in ev.key or "offsets_scan" in ev.key or "Memset" in ev.key:
                short = ev.key.split("jpeg_")[1].split("_kernel")[0] if "jpeg_" in ev.key \
                    else ev.key
                kern[short] = round(kern.get(short, 0) + ev.device_time_total / 1e3 / 5, 4)
        enc_ms, _ = time_ms(lambda: api_utils.encode_jpeg_batch(dev), iters)

        def host_clock(fn, k):
            fn()
            ts = []
            for _ in range(k):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            return float(np.median(ts))

        k = max(3, iters // 4)
        plan_ms = host_clock(lambda: je.EncodePlan([(h.shape, h.dtype) for h in host]), k)
        # the host part's largest piece: the files' bytes downloaded and made a bytes object
        d_files = torch.empty(sum(len(f) for f in files), dtype=torch.uint8, device="cuda")
        download_ms = host_clock(lambda: d_files.cpu().numpy().tobytes(), k)
        one_ms = host_clock(lambda: [enc(a) for a in host], k)
        with ThreadPoolExecutor(16) as pool:
            pool_ms = host_clock(lambda: list(pool.map(enc, host)), k)
        with tempfile.TemporaryDirectory() as tmp:
            def tail(fmt):
                outs = api_utils._unmold_overlay_file_batch(items, images, colors,
                                                            image_format=fmt)
                for b, o in enumerate(outs):
                    with open(os.path.join(tmp, f"{b}.{fmt}"), "wb") as f:
                        f.write(o[3])

            png_tail_ms = host_clock(lambda: tail("png"), k)
            jpeg_tail_ms = host_clock(lambda: tail("jpeg"), k)
        print(json.dumps({
            "workload": f"JPEG encode {name} overlays, quality 95 ({jpeg_mb:.1f} MB of files, "
                        f"{png_mb:.1f} MB as PNG)",
            "equal_to_cv2": same,
            "kernel_ms": kern, "kernel_ms_total": round(sum(kern.values()), 3),
            "api_utils_encode_jpeg_batch_ms": round(enc_ms, 3),
            "host_plan_ms": round(plan_ms, 3),
            "host_download_of_the_files_ms": round(download_ms, 3),
            "host_imencode_one_thread_ms": round(one_ms, 3),
            "host_imencode_16_threads_ms": round(pool_ms, 3),
            "do_inference_batch_tail_png_ms": round(png_tail_ms, 3),
            "do_inference_batch_tail_jpeg_ms": round(jpeg_tail_ms, 3),
            "host_threads": os.cpu_count(), **card()}), flush=True)


def annotate_case(iters):
    """The boxes, contour outlines and captions of display_instances drawn on the overlay
    (csrc/annotate.cu, DESIGN.md section 3.25) on 32 x 1024^2 x 100 and 16 x 2160x3840 x 50
    synthetic batches: the kernels of `UnmoldEngine.annotate` (pack, contour trace, draw,
    resolve) from a profile, the host caption stencils, and the tail of do_inference_batch (unmold
    + overlay + files written) with and without annotate, for PNG and JPEG.  The synthetic masks
    are thresholded noise: their outlines have thousands of segments each, far more than a real
    mask's."""
    import random
    import tempfile

    from torch.profiler import ProfilerActivity, profile

    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, visualize

    names = ["BG"] + ["class_%d" % i for i in range(1, 81)]
    for name, batch, hw, n in [("configs[1] 32 x 1024x1024 x 100", 32, (1024, 1024), 100),
                               ("configs[3] size: 16 x 2160x3840 x 50", 16, (2160, 3840), 50)]:
        ims = synth.make_batch(5, 4, hw, n, num_classes=81, max_instances=n)
        items = [(ims[b % 4].detections, ims[b % 4].mrcnn_mask, ims[b % 4].original_image_shape,
                  ims[b % 4].image_shape, ims[b % 4].window) for b in range(batch)]
        rng = np.random.default_rng(3)
        base = [synth.synth_rgb_image(rng, *hw) for _ in range(4)]
        images = [torch.from_numpy(base[b % 4]).cuda() for b in range(batch)]
        colors = visualize.random_colors(n, rng=random.Random(0))
        eng = UnmoldEngine(batch, n, (28, 28), 81)
        eng.plan([make_geom(*it[2:]) for it in items])
        d_det = torch.from_numpy(np.stack([it[0] for it in items])).cuda()
        d_msk = torch.from_numpy(np.stack([it[1] for it in items])).cuda()
        eng.enqueue(d_det, d_msk)
        stage = visualize.CompositeStage(eng, images, colors)
        stage.run()
        counts, boxes, ids, scs = eng.fetch_meta()
        boxes = [boxes[b, :int(counts[b])].copy() for b in range(batch)]
        ids = [ids[b, :int(counts[b])].copy() for b in range(batch)]
        scs = [scs[b, :int(counts[b])].copy() for b in range(batch)]
        hws = [hw] * batch

        def host_clock(fn, k):
            fn()
            ts = []
            for _ in range(k):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            return float(np.median(ts))

        k = max(3, iters // 4)
        caption_ms = host_clock(lambda: visualize.caption_stencils(boxes, hws, ids, names, scs), k)
        patches = visualize.caption_stencils(boxes, hws, ids, names, scs)
        rgb8 = np.stack([visualize.color_table(colors, n)] * batch)
        annotate = lambda: eng.annotate(stage.d_out, stage.d_off, rgb8, patches)   # noqa: E731
        annotate()
        d_vert, _, icoff = eng.trace_contours()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                annotate()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            for part, keys in (("pack", ("pack_",)), ("trace", ("contour_", "offsets_scan")),
                               ("draw", ("annotate_zero", "annotate_box", "annotate_vertex")),
                               ("resolve", ("annotate_resolve", "annotate_caption"))):
                if any(key in ev.key for key in keys):
                    kern[part] = round(kern.get(part, 0) + ev.device_time_total / 1e3 / 3, 4)
        step_ms = host_clock(annotate, k)
        with tempfile.TemporaryDirectory() as tmp:
            def tail(fmt, ann):
                outs = api_utils._unmold_overlay_file_batch(
                    items, images, colors, image_format=fmt, annotate=ann,
                    class_names=names if ann else None)
                for b, o in enumerate(outs):
                    with open(os.path.join(tmp, f"{b}.{fmt}"), "wb") as f:
                        f.write(o[3])

            tails = {f"do_inference_batch_tail_{fmt}{'_annotated' if ann else ''}_ms":
                     round(host_clock(lambda: tail(fmt, ann), k), 3)
                     for fmt in ("png", "jpeg") for ann in (False, True)}
        n_vert, n_contours = int(d_vert.shape[0]), int(icoff[-1])
        print(json.dumps({
            "workload": f"annotate {name} (synthetic noise masks)",
            "instances": int(sum(counts)), "contour_segments": n_vert - n_contours,
            "caption_patches": int(patches[0].shape[0]),
            "kernel_ms": kern, "annotate_step_ms_incl_host_reads": round(step_ms, 3),
            "host_caption_stencils_ms": round(caption_ms, 3), **tails, **card()}), flush=True)
        del eng, stage, d_det, d_msk
        torch.cuda.empty_cache()


def png_decode_case(iters):
    """PNG request bytes decoded on the device (csrc/png_decode.cu) against cv2.imdecode on the host,
    each followed by preprocess_input_batch: 32 x 1024^2 as cv2.imwrite writes them (level 1,
    Z_RLE, Sub rows), the same images at zlib level 6 (most other encoders' default), and
    16 x 2160x3840 as cv2.imwrite writes them.  Also the finder's candidates against the blocks
    chained, and the blocks the chain had to measure itself."""
    import zlib
    from concurrent.futures import ThreadPoolExecutor

    import cv2

    from torch.profiler import ProfilerActivity, profile

    from matterport_maskrcnn_with_tensorflow_serving_b200 import api_utils, png, serve

    def level6(rgb):
        raw = b"".join(b"\x01" + bytes(np.concatenate([r[:3], (r[3:].astype(np.int16) -
                                                               r[:-3]).astype(np.uint8)]))
                       for r in rgb.reshape(rgb.shape[0], -1))
        h, w = rgb.shape[:2]
        chunk = lambda t, d: (len(d).to_bytes(4, "big") + t + d +              # noqa: E731
                              zlib.crc32(t + d).to_bytes(4, "big"))
        ihdr = w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([8, 2, 0, 0, 0])
        return (png.SIGNATURE + chunk(b"IHDR", ihdr) + chunk(b"IDAT", zlib.compress(raw, 6)) +
                chunk(b"IEND", b""))

    rng = np.random.default_rng(13)
    m = Molder(api_utils.get_config())
    cv2_file = lambda a: cv2.imencode(".png", a[:, :, ::-1])[1].tobytes()   # noqa: E731
    for name, batch, hw, write in [("32 x 1024x1024 cv2.imwrite", 32, (1024, 1024), cv2_file),
                                   ("32 x 1024x1024 zlib level 6", 32, (1024, 1024), level6),
                                   ("configs[3] size: 16 x 2160x3840 cv2.imwrite", 16,
                                    (2160, 3840), cv2_file)]:
        base = [synth.synth_rgb_image(rng, *hw) for _ in range(4)]
        files = [write(a) for a in base]
        blobs = [files[b % 4] for b in range(batch)]
        mb = sum(len(b) for b in blobs) / 1e6
        m.decode_png_batch(blobs)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                m.decode_png_batch(blobs)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "png_" in ev.key:
                short = ev.key.split("png_")[1].split("_kernel")[0]
                kern[short] = round(kern.get(short, 0) + ev.device_time_total / 1e3 / 5, 4)
        plan = png.DecodePlan(blobs)
        sizes = [h * w * 3 for h, w, _ in plan.shapes]
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        out = torch.empty(int(off[-1]), dtype=torch.uint8, device="cuda")
        _, d_info, _ = m.png_decode_into(plan, out, off[:-1])
        info = d_info.cpu().numpy()
        nblk, seq, cand = info[:, 0], info[:, 1], info[:, 6]
        dec_ms, _ = time_ms(lambda: api_utils.decode_png_batch(blobs), iters)
        pre_ms, _ = time_ms(lambda: serve.preprocess_input_batch(blobs), iters)

        def host(pool):
            dec = (lambda b: cv2.cvtColor(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR),
                                          cv2.COLOR_BGR2RGB))
            arrs = list(pool.map(dec, blobs)) if pool else [dec(b) for b in blobs]
            return serve.preprocess_input_batch(arrs)

        def host_clock(fn, n):
            fn()
            ts = []
            for _ in range(n):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            return float(np.median(ts))

        one_ms = host_clock(lambda: host(None), max(3, iters // 4))
        with ThreadPoolExecutor(os.cpu_count()) as pool:
            pool_ms = host_clock(lambda: host(pool), max(3, iters // 4))
        print(json.dumps({
            "workload": f"PNG decode {name} ({mb:.1f} MB of files)",
            "kernel_ms": kern, "kernel_ms_total": round(sum(kern.values()), 3),
            "deflate_blocks_per_image_min_median_max": [int(nblk.min()), int(np.median(nblk)),
                                                        int(nblk.max())],
            "candidates_found_per_image_median": int(np.median(cand)),
            "blocks_measured_by_the_chain_per_image_median": int(np.median(seq)),
            "candidate_slots_per_tile": plan.K,
            "api_utils_decode_png_batch_ms": round(dec_ms, 3),
            "preprocess_input_batch_bytes_ms": round(pre_ms, 3),
            "host_imdecode_one_thread_then_preprocess_ms": round(one_ms, 3),
            "host_imdecode_pool_then_preprocess_ms": round(pool_ms, 3),
            "host_threads": os.cpu_count(), **card()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--only-eval", action="store_true", help="only the mask IoU / AP record")
    ap.add_argument("--only-cocoeval", action="store_true", help="only the COCO mask AP record")
    ap.add_argument("--only-bboxeval", action="store_true", help="only the COCO box AP record")
    ap.add_argument("--only-boundaryeval", action="store_true", help="only the Boundary AP "
                    "record")
    ap.add_argument("--only-polygons", action="store_true", help="only the polygon ground truth "
                    "record")
    ap.add_argument("--only-lvis", action="store_true", help="only the LVIS mask AP record")
    ap.add_argument("--only-jpeg", action="store_true", help="only the JPEG decode record")
    ap.add_argument("--only-png", action="store_true", help="only the PNG encode record")
    ap.add_argument("--only-jpeg-progressive", action="store_true",
                    help="only the progressive JPEG decode record")
    ap.add_argument("--only-png-decode", action="store_true", help="only the PNG decode record")
    ap.add_argument("--only-jpeg-encode", action="store_true", help="only the JPEG encode record")
    ap.add_argument("--only-annotate", action="store_true",
                    help="only the annotated overlay record")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    if args.only_annotate:
        annotate_case(args.iters)
        return
    if args.only_png_decode:
        png_decode_case(args.iters)
        return
    if args.only_jpeg_encode:
        jpeg_encode_case(args.iters)
        return
    if args.only_jpeg_progressive:
        jpeg_progressive_case(args.iters)
        return
    if args.only_png:
        png_case(args.iters)
        return
    if args.only_jpeg:
        jpeg_case(args.iters)
        return
    if args.only_cocoeval:
        cocoeval_case(args.iters)
        return
    if args.only_bboxeval:
        bboxeval_case(args.iters)
        return
    if args.only_boundaryeval:
        boundaryeval_case(args.iters)
        return
    if args.only_polygons:
        polygons_case(args.iters)
        return
    if args.only_lvis:
        lvis_case(args.iters)
        return
    eval_case(args.iters, args.cpu)
    if args.only_eval:
        return
    unmold_case("configs[1] 32 x 1024x1024 x 100", 32, (1024, 1024), 100, 81, 100, args.iters, composite=True)
    unmold_case("configs[2] 64 x 800x1333 (HxW) x U{1..100}", 64, (800, 1333), (1, 100), 81, 100,
                args.iters, base_images=16)
    unmold_case("configs[3] per-GPU shard: 16 x 2160x3840 x 50", 16, (2160, 3840), 50, 81, 50,
                args.iters, base_images=2)
    anchors_sweep(args.iters, args.cpu)
    mold_cases(args.iters, args.cpu)


if __name__ == "__main__":
    main()
