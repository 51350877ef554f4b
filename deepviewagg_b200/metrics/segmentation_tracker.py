"""SegmentationTracker of metrics/segmentation_tracker.py:11-108 on the GPU.

track() is one launch of ops.confusion_update on the model's output and labels: the argmax, the ignore mask and
the counting happen in the kernel, with no host copy and no host sync.  The reference recomputes acc, macc and
mIoU from the matrix after every batch; here they are computed from the same matrix when get_metrics() is
called, which gives the same values.  Loss meters, wandb and tensorboard are not part of this tracker."""
from typing import Any, Dict

from .confusion_matrix import ConfusionMatrix

IGNORE_LABEL = -1


class SegmentationTracker:
    def __init__(self, dataset, stage="train", wandb_log=False, use_tensorboard=False, ignore_label=IGNORE_LABEL):
        if wandb_log or use_tensorboard:
            raise NotImplementedError("SegmentationTracker: wandb and tensorboard logging are not supported")
        self._num_classes = dataset.num_classes
        self._ignore_label = ignore_label
        self._dataset = dataset
        self._n_iter = 0
        self.reset(stage)
        self._metric_func = {"miou": max, "macc": max, "acc": max, "loss": min, "map": max}

    def reset(self, stage="train"):
        self._stage = stage
        self._finalised = False
        self._confusion_matrix = ConfusionMatrix(self._num_classes)

    @property
    def confusion_matrix(self):
        """None until a batch with a label that is not ignored has been counted, as in the reference (which returns
        before counting a batch whose labels are all ignored)."""
        m = self._confusion_matrix.confusion_matrix
        return None if m is None or m.sum() == 0 else m

    def track(self, model, **kwargs):
        """Count the current batch: argmax of model.get_output() against model.get_labels()."""
        if not self._dataset.has_labels(self._stage):
            return
        if self._finalised:
            raise RuntimeError("Cannot track new values with a finalised tracker, you need to reset it first")
        outputs, labels = model.get_output(), model.get_labels()
        if labels.numel() == 0:
            return
        self._confusion_matrix.count_scores_batch(labels.detach(), outputs.detach(), ignore_label=self._ignore_label)

    def finalise(self, *args, **kwargs):
        self._finalised = True

    # the reference's attributes, computed from the matrix when read
    @property
    def _acc(self):
        return 100 * self._confusion_matrix.get_overall_accuracy()

    @property
    def _macc(self):
        return 100 * self._confusion_matrix.get_mean_class_accuracy()

    @property
    def _miou(self):
        return 100 * self._confusion_matrix.get_average_intersection_union()

    @property
    def _miou_per_class(self):
        if self.confusion_matrix is None:
            return {}
        return {i: "{:.2f}".format(100 * v)
                for i, v in enumerate(self._confusion_matrix.get_intersection_union_per_class()[0])}

    def get_metrics(self, verbose=False) -> Dict[str, Any]:
        metrics = {f"{self._stage}_acc": self._acc, f"{self._stage}_macc": self._macc,
                   f"{self._stage}_miou": self._miou}
        if verbose:
            metrics[f"{self._stage}_miou_per_class"] = self._miou_per_class
        return metrics

    @property
    def metric_func(self):
        return self._metric_func
