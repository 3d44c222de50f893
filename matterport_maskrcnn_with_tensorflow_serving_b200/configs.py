"""Stand-in for the reference's absent `configs` module (`import configs as cf`,
serve.py:22).  Attribute names are exactly the ones serve.py reads
(serve.py:78,114,120-136,165); values are deployment placeholders."""

HOST = "127.0.0.1"
gRPC_PORT = 8500
GRPC_TIMEOUT = 30.0
IMAGE_SIZE = 640                      # serve.py:114 -> cv2.resize to IMAGE_SIZE x IMAGE_SIZE
IN_TENSOR_IMAGE = "input_image"
IN_TENSOR_IMAGE_META = "input_image_meta"
IN_TENSOR_ANCHORS = "input_anchors"
IN_TENSOR_DTYPE = "float32"
MODEL_SIG_NAME = "serving_default"
MODEL_SPEC_NAME = "mask_rcnn"
OUT_TENSOR_DETECTION = "mrcnn_detection/Reshape_1"
OUT_DETECTION_SHAPE = (100, 6)        # serve.py:133 reshapes to (-1, *shape) -> [1,100,6]
OUT_TENSOR_MASK = "mrcnn_mask/Reshape_1"
OUT_MASK_SHAPE = (100, 28, 28, 81)    # serve.py:136
DAMAGE_CLASSES = ["class_%d" % i for i in range(1, 81)]
