"""`from model_configs import mconfig as mcf` (serve.py:23)."""
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from matterport_maskrcnn_with_tensorflow_serving_b200.model_configs import (  # noqa: E402,F401
    MaskRCNNServingConfig,
    mconfig,
)
