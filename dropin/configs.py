"""`import configs as cf` (serve.py:22): stand-in deployment constants."""
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from matterport_maskrcnn_with_tensorflow_serving_b200.configs import *  # noqa: E402,F401,F403
