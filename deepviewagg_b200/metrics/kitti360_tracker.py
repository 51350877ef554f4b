"""KITTI360Tracker of metrics/kitti360_tracker.py:25-368 with the current window's votes on the GPU.

The votes of the window being tracked (fp32 votes, int32 counts, claim stamps) live on the device and take one
ops.vote per sample.  When a sample of another window arrives, the table goes to the host, into the tracker's
temporary directory, as in the reference (holding every window in memory is what it avoids), and the other
window's table is loaded or created.  finalise() goes over every window: the vote confusion over the voted points
(ops.confusion_update with the counts as mask, ignored labels skipped) and, with full_res, the full-resolution
confusion through ops.full_res_predict(mode='own_votes'): a voted point keeps the argmax of its own votes, the
others take their nearest voted point (kitti360_tracker.py:219-222).

The dataset is duck-typed.  dataset.get_dataset(stage) gives the stage dataset with `windows` (names),
`window_raw_sizes` and `read_window(idx_window) -> (pos [N, 3], y [N] or None)`.  This last method is a
documented deviation: the reference calls read_kitti360_window on the window's PLY file, which is dataset code
outside this package.  A batch is split with data.to_data_list() when it has one (each element carrying
`idx_window`, `origin_id` and the `pred` rows set on the batch before the split, as in the reference), and is
one sample otherwise.

Differences from the reference: a duplicated origin id in one sample adds its last occurrence; an origin id
outside its window raises ValueError when the window is saved, not in track; a window without any vote has no
full-resolution prediction and raises ValueError with full_res (the reference interpolates from an empty set);
_make_submission and _zip_submission are not supported."""
import os
import os.path as osp
import tempfile
from typing import Any, Dict

import torch

from .. import ops
from .confusion_matrix import ConfusionMatrix, _status_message
from .s3dis_tracker import ORIGIN_ID_KEY
from .segmentation_tracker import SegmentationTracker


class KITTI360Tracker(SegmentationTracker):
    def reset(self, *args, **kwargs):
        super().reset(*args, **kwargs)
        self._vote_confusion_matrix = ConfusionMatrix(self._num_classes)
        self._full_confusion_matrix = ConfusionMatrix(self._num_classes)
        self._vote_miou = None
        self._full_vote_miou = None
        self._iou_per_class = {}
        self._vote_iou_per_class = {}
        self._full_vote_iou_per_class = {}
        self.windows = self.stage_dataset.windows
        self._temp_dir = None
        self._idx_window = None
        self._votes = self._counts = self._stamp = self._status = None

    @property
    def stage_dataset(self):
        return self._dataset.get_dataset(self._stage)

    @property
    def temp_dir(self):
        return None if self._temp_dir is None else self._temp_dir.name

    @property
    def has_labels(self):
        return self._dataset.has_labels(self._stage)

    def track(self, model, data=None, **kwargs):
        super().track(model)
        if self._stage == "train":
            return
        if self._temp_dir is None:
            self._temp_dir = tempfile.TemporaryDirectory()
        data = model.get_input() if data is None else data
        data = data.data if model.is_multimodal else data
        data.pred = model.get_output().detach()
        for d in (data.to_data_list() if hasattr(data, "to_data_list") else [data]):
            idx_window = d.idx_window
            if torch.is_tensor(idx_window):
                idx_window = int(idx_window.item())
            if idx_window != self._idx_window:
                self._save_window_tracking()
                self._load_window_tracking(idx_window, d.pred.device)
            origin = d[ORIGIN_ID_KEY]
            if origin is None:
                raise ValueError(f"The inputs given to the model do not have a {ORIGIN_ID_KEY} attribute.")
            origin = origin.flatten() if origin.dim() == 2 else origin
            ops.vote(self._votes, self._counts, self._stamp, origin.to(device=d.pred.device, dtype=torch.int64),
                     d.pred, status=self._status)

    def _window_path(self, idx_window):
        path = osp.join(self.temp_dir, self.windows[idx_window] + ".pt")
        os.makedirs(osp.dirname(path), exist_ok=True)
        return path

    def _save_window_tracking(self):
        if self._idx_window is None or self._idx_window < 0:
            return
        status = int(self._status.item())
        if status:
            raise ValueError(_status_message(status, self._num_classes))
        torch.save((self._votes.cpu(), self._counts.cpu()), self._window_path(self._idx_window))

    def _load_window_tracking(self, idx_window, device):
        path = self._window_path(idx_window)
        if osp.exists(path):
            votes, counts = torch.load(path)
        else:
            n = int(self.stage_dataset.window_raw_sizes[idx_window])
            votes = torch.zeros(n, self._num_classes, dtype=torch.float32)
            counts = torch.zeros(n, dtype=torch.int32)
        self._idx_window = idx_window
        self._votes = votes.to(device).contiguous()
        self._counts = counts.to(device).contiguous()
        self._stamp = torch.full((votes.shape[0],), -1, dtype=torch.int32, device=device)
        self._status = ops.eval_status(device)

    def finalise(self, full_res=False, make_submission=False, **kwargs):
        if make_submission and self._stage == "test":
            raise NotImplementedError("KITTI360Tracker: submissions are not supported")
        self._save_window_tracking()
        if self.has_labels:
            per_class_iou = self._confusion_matrix.get_intersection_union_per_class()[0]
            self._iou_per_class = {self._dataset.INV_OBJECT_LABEL[k]: v for k, v in enumerate(per_class_iou)}
        if self._stage == "train" or not self.has_labels or self._temp_dir is None:
            return
        device = self._votes.device
        vcm = self._vote_confusion_matrix._ensure(device)
        fcm = self._full_confusion_matrix._ensure(device) if full_res else None
        for idx_window in range(len(self.windows)):
            self._load_window_tracking(idx_window, device)
            pos, y = self.stage_dataset.read_window(idx_window)
            if y is None:
                continue
            y = y.to(device=device, dtype=torch.int64)
            ops.confusion_update(vcm, self._votes, y, ignore_label=self._ignore_label, counts=self._counts,
                                 status=self._vote_confusion_matrix.device_status)
            if full_res:
                ops.full_res_predict(self._votes, self._counts, pos.to(device), labels=y, cm=fcm,
                                     ignore_label=self._ignore_label, mode="own_votes",
                                     status=self._full_confusion_matrix.device_status)
        for cm, key in ((self._vote_confusion_matrix, "vote"), (self._full_confusion_matrix, "full_vote")):
            m = cm.confusion_matrix
            if m is not None and m.sum() > 0:
                setattr(self, f"_{key}_miou", cm.get_average_intersection_union() * 100)
                setattr(self, f"_{key}_iou_per_class", {self._dataset.INV_OBJECT_LABEL[k]: 100 * v
                                                        for k, v in enumerate(cm.get_intersection_union_per_class()[0])})

    def get_metrics(self, verbose=False) -> Dict[str, Any]:
        metrics = super().get_metrics(verbose)
        if verbose and self.has_labels:
            metrics[f"{self._stage}_iou"] = self._iou_per_class
        if self._vote_miou:
            metrics[f"{self._stage}_vote_miou"] = self._vote_miou
            if verbose:
                metrics[f"{self._stage}_vote_iou"] = self._vote_iou_per_class
        if self._full_vote_miou:
            metrics[f"{self._stage}_full_miou"] = self._full_vote_miou
            if verbose:
                metrics[f"{self._stage}_full_iou"] = self._full_vote_iou_per_class
        return metrics
