"""yolov5_obb_b200 — H100-native (sm_90a) engine behind yolov5_obb's hot-path entry points.

Only what the hot path needs lives here: csrc/ (CUDA kernels + the C ABI of include/y5obb.h) and the
host-side mirrors of the reference operator interfaces (nms_rotated, general, loss, yolo).
"""
__version__ = "0.1.0"
