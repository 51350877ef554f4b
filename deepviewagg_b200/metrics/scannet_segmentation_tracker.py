"""ScannetSegmentationTracker of metrics/scannet_segmentation_tracker.py:17-135 with its votes on the GPU.

The votes of every scan seen so far live in one device table (fp32 votes, int32 counts, claim stamps), each scan a
contiguous slice of it; a scan joins the table the first time it appears (dataset.get_raw_data(stage, id_scan,
remap_labels=True) gives its `pos` and `y`).  A track(full_res=True, data=...) call makes one ops.vote per sample
of the batch, its rows selected with elementwise ops over `data.batch` instead of boolean masks: no host sync when
`data.id_scan` is a CPU tensor (a CUDA id_scan is read back once per batch).
finalise(full_res=True) predicts every point of every scan with ops.full_res_predict(mode='interpolate_mean'): the
voted rows divided by their counts (the reference's in-place mean, taken in the kernel; the table keeps the sums),
then k = 1 interpolation and argmax, counted against the labels that are not `ignore_label`.

Differences from the reference: a duplicated origin id in one sample adds its last occurrence; an origin id
outside its scan raises ValueError at finalise; the DENSE layout and _make_submission are not supported."""
from typing import Any, Dict

import torch

from .. import _lib, ops
from .confusion_matrix import ConfusionMatrix, _status_message
from .s3dis_tracker import ORIGIN_ID_KEY
from .segmentation_tracker import SegmentationTracker


class ScannetSegmentationTracker(SegmentationTracker):
    def reset(self, stage="train"):
        super().reset(stage=stage)
        self._full_confusion_matrix = ConfusionMatrix(self._num_classes)
        self._raw_datas = {}
        self._scan_slices = {}      # id_scan -> (start, stop) rows of the vote table
        self._votes = self._vote_counts = self._stamp = self._status = None
        self._full_preds = {}
        self._full_acc = None

    def track(self, model, full_res=False, **kwargs):
        super().track(model)
        self._conv_type = getattr(model, "conv_type", None)
        if not full_res or self._stage == "train" or kwargs.get("data") is None:
            return
        data = kwargs["data"]
        data = data.data if model.is_multimodal else data
        self._vote(data, model.get_output().detach())

    def _add_scan(self, id_scan, device):
        raw = self._dataset.get_raw_data(self._stage, id_scan, remap_labels=True)
        self._raw_datas[id_scan] = raw
        n, K = raw.pos.shape[0], self._num_classes
        start = 0 if self._votes is None else self._votes.shape[0]
        self._scan_slices[id_scan] = (start, start + n)
        new = (torch.zeros((n, K), dtype=torch.float32, device=device), torch.zeros(n, dtype=torch.int32, device=device),
               torch.full((n,), -1, dtype=torch.int32, device=device))
        if self._votes is None:
            self._votes, self._vote_counts, self._stamp = new
            self._status = ops.eval_status(device)
        else:
            self._votes = torch.cat([self._votes, new[0]])
            self._vote_counts = torch.cat([self._vote_counts, new[1]])
            self._stamp = torch.cat([self._stamp, new[2]])

    def _vote(self, data, output):
        if self._conv_type == "DENSE":
            raise NotImplementedError("ScannetSegmentationTracker: the DENSE layout is not supported")
        id_scans = data.id_scan
        if id_scans.dim() > 1:
            id_scans = id_scans.squeeze()
        id_scans = [int(i) for i in id_scans.reshape(-1).tolist()]
        for id_scan in id_scans:
            if id_scan not in self._raw_datas:
                self._add_scan(id_scan, output.device)
        origin = data[ORIGIN_ID_KEY].to(device=output.device, dtype=torch.int64).reshape(-1)
        batch = data.batch.to(output.device).reshape(-1)
        # one vote per sample, as the reference adds sample after sample (an id in two samples counts twice): the
        # sample's rows go to the start of its scan + origin id, every other row to -1, which the kernel skips (its
        # flag goes to a scratch word); an origin id outside its scan is flagged in the table's status word
        scratch = ops.eval_status(output.device)
        for b, id_scan in enumerate(id_scans):
            start, stop = self._scan_slices[id_scan]
            mine = batch == b
            inside = (origin >= 0) & (origin < stop - start)
            row = torch.where(mine & inside, origin + start, -1)
            ops.vote(self._votes, self._vote_counts, self._stamp, row, output, status=scratch)
            self._status |= (mine & ~inside).any().int() * _lib.DVA_EVAL_BAD_ID

    def _predict_full_res(self):
        status = int(self._status.item()) if self._status is not None else 0
        if status:
            raise ValueError(_status_message(status, self._num_classes))
        cm = self._full_confusion_matrix._ensure(self._votes.device) if self._dataset.has_labels(self._stage) else None
        for id_scan, (start, stop) in self._scan_slices.items():
            raw = self._raw_datas[id_scan]
            labels = raw.y.to(device=self._votes.device, dtype=torch.int64) if cm is not None else None
            pred, _ = ops.full_res_predict(self._votes[start:stop], self._vote_counts[start:stop],
                                           raw.pos.to(self._votes.device), labels=labels, cm=cm,
                                           ignore_label=self._ignore_label, mode="interpolate_mean",
                                           status=self._full_confusion_matrix.device_status)
            self._full_preds[id_scan] = pred

    def finalise(self, full_res=False, make_submission=False, **kwargs):
        if make_submission:
            raise NotImplementedError("ScannetSegmentationTracker: _make_submission is not supported")
        if not full_res or self._votes is None:
            return
        self._predict_full_res()
        if self._dataset.has_labels(self._stage):
            c = self._full_confusion_matrix
            self._full_acc = 100 * c.get_overall_accuracy()
            self._full_macc = 100 * c.get_mean_class_accuracy()
            self._full_miou = 100 * c.get_average_intersection_union()

    def get_metrics(self, verbose=False) -> Dict[str, Any]:
        metrics = super().get_metrics(verbose)
        if self._full_acc:
            metrics[f"{self._stage}_full_acc"] = self._full_acc
            metrics[f"{self._stage}_full_macc"] = self._full_macc
            metrics[f"{self._stage}_full_miou"] = self._full_miou
        return metrics
