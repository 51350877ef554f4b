"""S3DISTracker of metrics/s3dis_tracker.py:15-139 with the test area's votes on the GPU.

The vote table of the test area (fp32 votes [N, K], int32 counts [N]) lives on the model's device; every
track(full_res=True) call is one ops.vote (two launches, no host sync).  finalise() computes
  * the vote confusion over the voted points (ops.confusion_update with the counts as mask), and
  * the full-resolution confusion through ops.full_res_predict: the nearest voted point of every point of the
    area (mapping.knn_query) and the fused k = 1 knn_interpolate + argmax + confusion kernel.

Deliberate differences from the reference:
  * a duplicated origin id in one batch adds its last occurrence (the reference's index_put_ leaves it
    undefined);
  * an origin id outside the area raises ValueError at the first metric read, not inside track (the
    reference's originids.max() is a host sync per batch);
  * ties in the nearest-neighbour search go to the lower voted index (torch_cluster's order is undocumented);
  * ply_output is not supported."""
from typing import Any, Dict

import torch

from .. import ops
from .confusion_matrix import ConfusionMatrix, _status_message
from .segmentation_tracker import SegmentationTracker

ORIGIN_ID_KEY = "origin_id"     # SaveOriginalPosId.KEY


class _VoteTable:
    """Votes, counts, claim stamps and positions / labels of one area, on one device."""

    def __init__(self, pos, y, num_classes, device):
        n = pos.shape[0]
        self.pos = pos.to(device=device, dtype=torch.float32).contiguous()
        self.y = y.to(device=device, dtype=torch.int64).contiguous()
        self.votes = torch.zeros((n, num_classes), dtype=torch.float32, device=device)
        self.prediction_count = torch.zeros(n, dtype=torch.int32, device=device)
        self.stamp = torch.full((n,), -1, dtype=torch.int32, device=device)
        self.status = ops.eval_status(device)

    def add(self, ids, outputs):
        ops.vote(self.votes, self.prediction_count, self.stamp, ids, outputs, status=self.status)

    def check(self):
        status = int(self.status.item())
        if status:
            raise ValueError(_status_message(status, self.votes.shape[1]))


class S3DISTracker(SegmentationTracker):
    def reset(self, *args, **kwargs):
        super().reset(*args, **kwargs)
        self._test_area = None
        self._full_vote_miou = None
        self._vote_miou = None
        self._full_confusion = None
        self._iou_per_class = {}

    def track(self, model, full_res=False, data=None, **kwargs):
        super().track(model)
        if self._stage == "train" or not full_res:
            return
        if self._test_area is None:
            area = self._dataset.test_data
            if getattr(area, "y", None) is None:
                raise ValueError("It seems that the test area data does not have labels (attribute y).")
            self._test_area = _VoteTable(area.pos, area.y, self._num_classes, model.get_output().device)
        inputs = data if data is not None else model.get_input()
        originids = inputs.data[ORIGIN_ID_KEY] if model.is_multimodal else inputs[ORIGIN_ID_KEY]
        if originids is None:
            raise ValueError(f"The inputs given to the model do not have a {ORIGIN_ID_KEY} attribute.")
        if originids.dim() == 2:
            originids = originids.flatten()
        outputs = model.get_output().detach()
        self._test_area.add(originids.to(device=outputs.device, dtype=torch.int64), outputs)

    def finalise(self, full_res=False, vote_miou=True, ply_output="", **kwargs):
        if ply_output:
            raise NotImplementedError("S3DISTracker: ply_output is not supported")
        per_class_iou = self._confusion_matrix.get_intersection_union_per_class()[0]
        self._iou_per_class = {self._dataset.INV_OBJECT_LABEL[k]: v for k, v in enumerate(per_class_iou)}
        if self._test_area is None:
            return
        self._test_area.check()
        area = self._test_area
        if vote_miou:
            c = ConfusionMatrix(self._num_classes)
            c.count_scores_batch(area.y, area.votes, counts=area.prediction_count)
            self._vote_miou = c.get_average_intersection_union() * 100
            self._vote_iou_per_class = {self._dataset.INV_OBJECT_LABEL[k]: 100 * v
                                        for k, v in enumerate(c.get_intersection_union_per_class()[0])}
        if full_res:
            self._compute_full_miou()

    def _compute_full_miou(self):
        if self._full_vote_miou is not None:
            return
        area = self._test_area
        self._full_confusion = ConfusionMatrix(self._num_classes)
        cm = self._full_confusion._ensure(area.votes.device)
        ops.full_res_predict(area.votes, area.prediction_count, area.pos, labels=area.y, cm=cm,
                             mode="interpolate", status=self._full_confusion.device_status)
        self._full_vote_miou = self._full_confusion.get_average_intersection_union() * 100
        self._full_vote_iou_per_class = {self._dataset.INV_OBJECT_LABEL[k]: 100 * v
                                         for k, v in enumerate(self._full_confusion.get_intersection_union_per_class()[0])}

    @property
    def full_confusion_matrix(self):
        return self._full_confusion

    def get_metrics(self, verbose=False) -> Dict[str, Any]:
        metrics = super().get_metrics(verbose)
        if verbose:
            metrics[f"{self._stage}_iou"] = self._iou_per_class
        if self._full_vote_miou:
            metrics[f"{self._stage}_full_vote_miou"] = self._full_vote_miou
            metrics[f"{self._stage}_full_vote_iou"] = self._full_vote_iou_per_class
        if self._vote_miou:
            metrics[f"{self._stage}_vote_miou"] = self._vote_miou
            metrics[f"{self._stage}_vote_iou"] = self._vote_iou_per_class
        return metrics
