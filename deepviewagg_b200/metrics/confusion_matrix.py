"""ConfusionMatrix of metrics/confusion_matrix.py:6-97 with its counts on the GPU.

The counts are an int64 [K, K] tensor on the device (row = ground truth, column = prediction), updated in place by
ops.confusion_update: no host copy and no host sync per batch.  The metric methods copy the matrix to the host
once per update and apply the reference's float64 numpy formulas to it, so they return the same floats.

A label or prediction outside [0, K) is not counted; it sets a bit of the device status word, and the first read
of the matrix raises ValueError (the reference asserts on the prediction inside count_predicted_batch, which
needs a host sync per batch)."""
import numpy as np
import torch

from .. import _lib, ops


class ConfusionMatrix:
    def __init__(self, number_of_labels=2, device=None):
        self.number_of_labels = int(number_of_labels)
        self._device = None if device is None else torch.device(device)
        self._counts = None    # int64 [K, K] on the device, created with the first batch
        self._status = None    # int32 [1] on the device
        self._host = None      # numpy copy of _counts, valid until the next update

    @staticmethod
    def create_from_matrix(confusion_matrix):
        cm = np.asarray(confusion_matrix)
        if cm.ndim != 2 or cm.shape[0] != cm.shape[1]:
            raise ValueError("create_from_matrix: the matrix must be square")
        matrix = ConfusionMatrix(cm.shape[0])
        matrix._host = cm.astype(np.int64)
        return matrix

    # ---- device side
    def _ensure(self, device):
        if self._counts is None:
            device = self._device if self._device is not None else device
            K = self.number_of_labels
            self._counts = torch.zeros((K, K), dtype=torch.int64, device=device)
            self._status = ops.eval_status(device)
            if self._host is not None:      # created from a host matrix: continue counting from it
                self._counts.copy_(torch.from_numpy(self._host))
        self._host = None
        return self._counts

    @property
    def device_counts(self):
        """The int64 [K, K] counts on the device (None before the first batch)."""
        return self._counts

    @property
    def device_status(self):
        return self._status

    def _to_device(self, t):
        if isinstance(t, np.ndarray):
            t = torch.from_numpy(t)
        if not t.is_cuda:
            dev = self._device or (self._counts.device if self._counts is not None else torch.device("cuda"))
            t = t.to(dev)
        return t.long() if t.dtype != torch.int64 else t

    def count_predicted_batch(self, ground_truth_vec, predicted):
        """Add a batch of (ground truth, prediction) pairs; CUDA tensors stay where they are, numpy arrays and CPU
        tensors are copied to the device once."""
        gt = self._to_device(ground_truth_vec).reshape(-1)
        pred = self._to_device(predicted).reshape(-1)
        cm = self._ensure(gt.device)
        ops.confusion_update(cm, pred, gt, status=self._status)

    def count_scores_batch(self, ground_truth_vec, scores, ignore_label=None, counts=None):
        """Add argmax(scores, 1) against the ground truth in one launch, skipping `ignore_label` and, with
        counts, the rows whose count is 0 (the tracker's per-batch update)."""
        cm = self._ensure(scores.device)
        ops.confusion_update(cm, scores, ground_truth_vec, ignore_label=ignore_label, counts=counts,
                             status=self._status)

    # ---- host side: the reference's formulas on the numpy matrix
    @property
    def confusion_matrix(self):
        """The K x K numpy int64 array (None before the first batch, as in the reference)."""
        if self._host is None and self._counts is not None:
            status = int(self._status.item())
            if status:
                raise ValueError(_status_message(status, self.number_of_labels))
            self._host = self._counts.cpu().numpy()
        return self._host

    def get_count(self, ground_truth, predicted):
        return self.confusion_matrix[ground_truth][predicted]

    def get_confusion_matrix(self):
        return self.confusion_matrix

    def _matrix(self):
        cm = self.confusion_matrix
        return np.zeros((self.number_of_labels,) * 2, dtype=np.int64) if cm is None else cm

    def get_intersection_union_per_class(self):
        """(iou, existing_class_mask): iou = 1e-8 + TP / (union + 1e-8), a class exists when union > 1e-3."""
        cm = self._matrix()
        tp = np.diagonal(cm)
        union = np.sum(cm, axis=0) + np.sum(cm, axis=1) - tp
        return 1e-8 + tp / (union + 1e-8), union > 1e-3

    def get_overall_accuracy(self):
        cm = self._matrix()
        total = int(cm.sum())
        return float(int(np.trace(cm))) / (total if total != 0 else 1)

    def get_average_intersection_union(self, missing_as_one=False):
        values, existing = self.get_intersection_union_per_class()
        if np.sum(existing) == 0:
            return 0
        if missing_as_one:
            values[~existing] = 1
            existing[:] = True
        return np.sum(values[existing]) / np.sum(existing)

    def get_mean_class_accuracy(self):
        cm = self._matrix()
        acc, present = 0, 0
        for i in range(self.number_of_labels):   # class order: the float sum of the reference
            total = np.sum(cm[i, :])
            if total:
                present += 1
                acc = acc + cm[i][i] / max(1, total)
        return 0 if present == 0 else acc / present

    def count_gt(self, ground_truth):
        return self._matrix()[ground_truth, :].sum()


def _status_message(status, K):
    what = []
    if status & _lib.DVA_EVAL_BAD_LABEL:
        what.append(f"a label outside [0, {K}) that is not the ignore label")
    if status & _lib.DVA_EVAL_BAD_PRED:
        what.append(f"a prediction outside [0, {K})")
    if status & _lib.DVA_EVAL_BAD_ID:
        what.append("an origin id outside the vote table")
    return "segmentation metrics: the tracked batches held " + " and ".join(what)
