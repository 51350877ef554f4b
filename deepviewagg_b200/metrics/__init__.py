"""Segmentation metrics on the GPU with the API of the reference's torch_points3d/metrics: the confusion matrix
and the trackers keep their counts and vote tables on the device and update them with the kernels of
libdva_eval.so (include/dva_eval.h)."""
from .confusion_matrix import ConfusionMatrix
from .segmentation_tracker import SegmentationTracker
from .s3dis_tracker import S3DISTracker
from .scannet_segmentation_tracker import ScannetSegmentationTracker
from .kitti360_tracker import KITTI360Tracker

__all__ = ["ConfusionMatrix", "SegmentationTracker", "S3DISTracker", "ScannetSegmentationTracker", "KITTI360Tracker"]
