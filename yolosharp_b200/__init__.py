"""yolosharp_b200: H100-native (sm_90a) YOLO forward + NMS engine behind the YoloSharp interface.

The product is the C-ABI shared library `lib/libyolob200.so` (sources in `csrc/`, header in
`include/yolob200.h`); this package is its host-side mirror of the reference's operator surface.
"""
from ._build import build  # noqa: F401
from ._lib import YbError  # noqa: F401
from .api import Config, Detector, Ops, Segmenter, YoloResult, YoloTask, Yolov8, Yolov8Segment, Yolov11  # noqa: F401
from .engine import Comm, Engine, adamw_step, conv_backward, conv_forward, bn_silu_backward, bn_silu_train_forward, detection_loss, masks, nms  # noqa: F401
