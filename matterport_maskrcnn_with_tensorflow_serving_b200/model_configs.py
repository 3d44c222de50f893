"""Stand-in for the reference's absent `model_configs` module
(`from model_configs import mconfig as mcf`, serve.py:23).

serve.py reads IMAGE_MIN_DIM, IMAGE_MIN_SCALE, IMAGE_MAX_DIM, IMAGE_RESIZE_MODE
(serve.py:93-96), NUM_CLASSES (:102) and, through `mold_image(..., mcf)` (:98),
MEAN_PIXEL; `get_anchors` needs the RPN_* / BACKBONE_* entries.  The reference's actual
values are not in its tree, so these are the public matterport/Mask_RCNN
`mrcnn/config.py` defaults; every kernel takes them as parameters, none are compiled in.
"""
import numpy as np


class MaskRCNNServingConfig:
    BACKBONE = "resnet101"
    BACKBONE_STRIDES = [4, 8, 16, 32, 64]
    RPN_ANCHOR_SCALES = (32, 64, 128, 256, 512)
    RPN_ANCHOR_RATIOS = [0.5, 1, 2]
    RPN_ANCHOR_STRIDE = 1
    IMAGE_RESIZE_MODE = "square"
    IMAGE_MIN_DIM = 800
    IMAGE_MAX_DIM = 1024
    IMAGE_MIN_SCALE = 0
    MEAN_PIXEL = np.array([123.7, 116.8, 103.9])
    NUM_CLASSES = 81
    MASK_SHAPE = [28, 28]
    DETECTION_MAX_INSTANCES = 100


mconfig = MaskRCNNServingConfig()
