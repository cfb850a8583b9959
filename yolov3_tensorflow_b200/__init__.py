"""yolov3_tensorflow_b200 — the YOLOv3 hot path of wizyoung/YOLOv3_TensorFlow
(model.yolov3.forward/predict, utils.nms_utils.gpu_nms, the darknet weight loader) on
hand-written sm_90a CUDA kernels behind a C ABI (libyolob200.so, include/yolob200.h).

Importing the package loads the shared library; it fails loudly if it has not been built.
"""
from . import _lib  # noqa: F401  (raises ImportError when libyolob200.so is missing)
from .model import yolov3  # noqa: F401
from .utils.nms_utils import gpu_nms, batched_gpu_nms, cpu_nms, py_nms  # noqa: F401
from .utils.misc_utils import (load_weights, parse_anchors, read_class_names, config_learning_rate,  # noqa: F401
                               config_optimizer, learning_rate_at, save_checkpoint, restore_checkpoint)

__version__ = "0.1.0"
