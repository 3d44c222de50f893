"""H100-native (sm_90a) implementation of the CPU-side serving hot path of
huyhoang17/matterport-maskrcnn-with-tensorflow-serving: `api_utils.get_anchors`,
`api_utils.unmold_detections` and the `preprocess_input` mold step, behind the
reference's own Python signatures.  See DESIGN.md / INTEGRATION.md.

Importing the package does not touch the GPU; the first call loads lib/libmrx.so and
raises if it (or a CUDA device) is missing -- there is no CPU fallback.
"""
from . import api_utils, configs, model_configs, synth  # noqa: F401
from .api_utils import get_anchors, unmold_detections, unmold_detections_batch  # noqa: F401

__all__ = ["api_utils", "configs", "model_configs", "synth", "get_anchors",
           "unmold_detections", "unmold_detections_batch"]
