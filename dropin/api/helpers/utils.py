"""`from api.helpers import utils as api_utils` (serve.py:21) resolved to the
H100 implementation.  Put the `dropin/` directory on PYTHONPATH ahead of the original app."""
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from matterport_maskrcnn_with_tensorflow_serving_b200.api_utils import (  # noqa: E402,F401
    get_anchors,
    get_config,
    load_img,
    set_config,
    unmold_detections,
    unmold_detections_batch,
)
