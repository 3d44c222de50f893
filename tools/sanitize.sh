#!/bin/bash
# compute-sanitizer over small parity tests of every kernel family (the team kernel synchronises
# through named barriers, shared-memory atomics and bulk async copies; the packed-expand and RLE
# kernels through warp-level primitives and bulk copies; the contour and RLE-string kernels through
# warp shuffles and CTA scans; the mask IoU and match kernels through warp shuffles and word loads
# realigned across plane boundaries, the COCO match kernel also through a shared-memory bitmask
# (with mask and with box areas, the box IoU kernel reading the kept boxes);
# the polygon kernels through CTA scans and the band transpose they share with the RLE decode;
# the boundary kernel through a CTA barrier between its two passes and warp-synchronous rows in
# shared memory, the boundary IoU kernel through the pair walk; the LVIS rank kernel through the
# CTA barrier between its category and counting passes and the status table it reads; the JPEG
# kernels through CTA scans of the unstuffed scan, the shared-memory sync rounds of the Huffman
# decode, the walk across CTAs and the warp-synchronous IDCT; the PNG kernels through CTA scans of
# the tile passes, shared-memory histograms, word atomics on the bit stream and the per-chunk CRC
# combine across a warp).
# Run on a GPU box:
#   bash tools/sanitize.sh   -> build/sanitizer_<tool>.log
cd "$(dirname "$0")/.."
mkdir -p build
SEL="expand_launches_after_one_prepare or mixed_geometries_in_one_launch or more_instances or every_box or no_detections or small_boxes or chunk_size or leading_unit or (packed_masks and (hw0 or hw1 or hw2 or hw7 or hw8)) or packed_batch_ragged or (rle_equals and not hw4 and not hw5) or rle_touching or all_zero_box or composite_on_device or out_of_range or alpha_sweep or (production_kernel and (small_mixed or tiny_boxes)) or identity_resize or byte_canvas_after or (contours_equal_oracle and not hw4 and not hw5) or mixed_shapes_and_an_empty or packed_routes or mask_contours_numpy_entry or (rle_strings_equal and float32 and not hw4 and not hw5) or rle_strings_touching or rle_strings_batch_of_empty or (ap_equals_oracle_small_shapes and (hw0 or hw2)) or mixed_shapes_no_predictions or duplicate_and_empty_ground_truth or evaluate_drop_ins or stream_equals_oracle or add_results_equals or (random_polygons_equal_oracle and (hw1 or hw4)) or known_answers or mixed_batches_equal or box_ious_equal_bbiou or add_results_equals_oracle or one_unmold_for_both or (ground_truth_boundaries_equal_cv2 and 0.02) or (prediction_boundaries_equal_cv2 and 0.5) or (add_batch_equals_oracle and 0.005) or one_unmold_for_three or (lvis_ranks_equal and (seed2 or seed4)) or lvis_and_coco_evaluators or coefficients_equal_the_oracle or results_do_not_depend_on_S or exif_orientations or corrupt_data_raises or device_intermediates_equal_the_oracle"
for tool in memcheck synccheck racecheck; do
  echo "== $tool"
  timeout 600 compute-sanitizer --tool $tool --error-exitcode 9 \
    python -m pytest tests/test_gpu_unmold.py tests/test_gpu_pack.py tests/test_gpu_rle.py tests/test_gpu_composite.py \
    tests/test_gpu_contours.py tests/test_gpu_kernel_paths.py tests/test_gpu_coco.py tests/test_gpu_eval.py \
    tests/test_gpu_cocoeval.py tests/test_gpu_polygons.py tests/test_gpu_cocoeval_bbox.py tests/test_gpu_cocoeval_boundary.py \
    tests/test_gpu_lvis.py tests/test_gpu_jpeg.py tests/test_gpu_png.py -q -x -k "$SEL" > build/sanitizer_$tool.log 2>&1
  echo "exit $?"
  tail -3 build/sanitizer_$tool.log
done
