"""CPU oracle for the Mask R-CNN serving hot path.  TEST INFRASTRUCTURE ONLY.

This package is a NumPy/SciPy restatement of the algorithm that the reference's
`serve.py` reaches through `api_utils.get_anchors` (serve.py:105),
`api_utils.unmold_detections` (serve.py:147-154) and the body of
`preprocess_input` (serve.py:83-107).  Those function bodies are not vendored in
the reference repository (serve.py:17-23 import them from un-vendored, un-pinned packages:
a fork of matterport/Mask_RCNN, scikit-image, scipy), so:

    *** PARITY UNPINNED ***  The reference ships no tests, golden vectors or
    fixtures for this path and its implementation cannot be imported here.  The
    oracle follows the published matterport/Mask_RCNN `mrcnn/model.py`,
    `mrcnn/utils.py`, `mrcnn/config.py` and scikit-image >= 0.19
    `transform.resize` (which executes `scipy.ndimage.zoom(..., order=1,
    mode='grid-constant', cval=0, grid_mode=True)`).  `cv2.resize`
    (serve.py:89) is the one step whose real implementation is importable, and
    the mold oracle calls the real cv2.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu-baseline /
`--impl reference` legs may import this package.  The product package
(`matterport_maskrcnn_with_tensorflow_serving_b200`) never does.
"""
from .mrcnn_oracle import (  # noqa: F401
    OracleConfig,
    norm_boxes,
    denorm_boxes,
    resize,
    resize_explicit,
    unmold_mask,
    unmold_detections,
    compute_backbone_shapes,
    generate_anchors,
    generate_pyramid_anchors,
    get_anchors,
    resize_image,
    mold_image,
    compose_image_meta,
    preprocess_input,
    random_colors,
    apply_mask,
    composite_instances,
    rle_encode,
    rle_decode,
)
