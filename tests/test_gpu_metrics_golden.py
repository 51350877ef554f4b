"""The GPU trackers reproduce the fixtures made by executing the reference's trackers
(oracle/make_golden_metrics.py): confusion matrices as integers, every get_metrics value as float64 and
full-resolution predictions element for element."""
import json
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from deepviewagg_b200.metrics import KITTI360Tracker, S3DISTracker, ScannetSegmentationTracker, SegmentationTracker

pytestmark = pytest.mark.gpu
K = 6


def fixture(name):
    z = np.load(os.path.join(GOLDEN, f"metrics_{name}.npz"), allow_pickle=False)
    return {k: z[k] for k in z.files}, json.loads(str(z["metrics"]))


def same_metrics(got, want):
    def conv(v):
        return {str(k): conv(x) for k, x in v.items()} if isinstance(v, dict) else (v if isinstance(v, str) else float(v))
    assert {k: conv(v) for k, v in got.items()} == want


class Dataset:
    def __init__(self, **kw):
        self.num_classes = K
        self.INV_OBJECT_LABEL = {i: f"c{i}" for i in range(K)}
        self.__dict__.update(kw)

    def has_labels(self, stage):
        return True


class Model:
    def __init__(self, out, y, inp=None, multimodal=False):
        self.out, self.y, self.inp, self.is_multimodal = out, y, inp, multimodal

    def get_output(self):
        return self.out

    def get_labels(self):
        return self.y

    def get_input(self):
        return self.inp


class Sample(dict):
    """Attribute and item access, as torch_geometric's Data gives (a missing attribute is an AttributeError)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None

    def __setattr__(self, k, v):
        self[k] = v


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_segmentation_tracker():
    z, want = fixture("segmentation")
    tr = SegmentationTracker(Dataset(), stage="val")
    for s, y in zip(z["scores"], z["labels"]):
        tr.track(Model(cu(s), cu(y)))
    assert (tr.confusion_matrix == z["cm"]).all()
    same_metrics(tr.get_metrics(verbose=True), want)


def test_all_ignored_batches_leave_no_matrix():
    tr = SegmentationTracker(Dataset(), stage="val")
    tr.track(Model(torch.randn(5, K, device="cuda"), torch.full((5,), -1, device="cuda")))
    assert tr.confusion_matrix is None
    assert tr.get_metrics(verbose=True)["val_miou_per_class"] == {}


def test_s3dis_tracker():
    z, want = fixture("s3dis")
    area = types.SimpleNamespace(pos=torch.from_numpy(z["pos"]), y=torch.from_numpy(z["y"]))
    tr = S3DISTracker(Dataset(test_data=area), stage="test")
    for b, (ids, s, lab) in enumerate(zip(z["ids"], z["scores"], z["labels"])):
        if b % 2:      # a multimodal input: the origin ids are read from inputs.data
            model = Model(cu(s), cu(lab), types.SimpleNamespace(data={"origin_id": cu(ids)}), multimodal=True)
        else:
            model = Model(cu(s), cu(lab), {"origin_id": cu(ids)})
        tr.track(model, full_res=True)
    tr.finalise(full_res=True, vote_miou=True)
    assert (tr.confusion_matrix == z["cm"]).all()
    assert (tr.full_confusion_matrix.confusion_matrix == z["full_cm"]).all()
    same_metrics(tr.get_metrics(verbose=True), want)


def test_scannet_tracker():
    z, want = fixture("scannet")
    ds = Dataset()
    ds.get_raw_data = lambda stage, i, remap_labels=True: types.SimpleNamespace(
        pos=torch.from_numpy(z[f"pos{i}"]), y=torch.from_numpy(z[f"y{i}"]))
    tr = ScannetSegmentationTracker(ds, stage="val")
    b = 0
    while f"b{b}/id_scan" in z:
        data = Sample(id_scan=torch.from_numpy(z[f"b{b}/id_scan"]), batch=cu(z[f"b{b}/batch"]),
                      origin_id=cu(z[f"b{b}/origin_id"]))
        tr.track(Model(cu(z[f"b{b}/scores"]), cu(z[f"b{b}/labels"])), full_res=True, data=data)
        b += 1
    tr.finalise(full_res=True)
    assert (tr.confusion_matrix == z["cm"]).all()
    assert (tr._full_confusion_matrix.confusion_matrix == z["full_cm"]).all()
    for s in (0, 1):
        assert torch.equal(tr._full_preds[s].cpu(), torch.from_numpy(z[f"full_pred{s}"]))
    same_metrics(tr.get_metrics(verbose=True), want)


def test_scannet_track_does_not_sync():
    z, _ = fixture("scannet")
    ds = Dataset()
    ds.get_raw_data = lambda stage, i, remap_labels=True: types.SimpleNamespace(
        pos=torch.from_numpy(z[f"pos{i}"]), y=torch.from_numpy(z[f"y{i}"]))
    tr = ScannetSegmentationTracker(ds, stage="val")
    batches = []
    for b in range(3):
        data = Sample(id_scan=torch.from_numpy(z[f"b{b}/id_scan"]), batch=cu(z[f"b{b}/batch"]),
                      origin_id=cu(z[f"b{b}/origin_id"]))
        batches.append((Model(cu(z[f"b{b}/scores"]), cu(z[f"b{b}/labels"])), data))
    tr.track(batches[0][0], full_res=True, data=batches[0][1])     # both scans join the table here
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for model, data in batches[1:]:
            tr.track(model, full_res=True, data=data)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_kitti360_tracker_with_window_switches():
    z, want = fixture("kitti360")
    windows = [f"seq_0/w{i}" for i in range(3)]
    sizes = [z[f"pos{w}"].shape[0] for w in range(3)]
    stage = types.SimpleNamespace(windows=windows, window_raw_sizes=sizes,
                                  read_window=lambda w: (torch.from_numpy(z[f"pos{w}"]), torch.from_numpy(z[f"y{w}"])))
    ds = Dataset()
    ds.get_dataset = lambda s: stage
    tr = KITTI360Tracker(ds, stage="val")
    for i, w in enumerate(z["order"]):
        data = Sample(idx_window=int(w), origin_id=cu(z[f"s{i}/ids"]))
        tr.track(Model(cu(z[f"s{i}/scores"]), cu(z[f"s{i}/labels"])), data=data)
    tr.finalise(full_res=True)
    assert (tr.confusion_matrix == z["cm"]).all()
    assert (tr._vote_confusion_matrix.confusion_matrix == z["vote_cm"]).all()
    assert (tr._full_confusion_matrix.confusion_matrix == z["full_cm"]).all()
    same_metrics(tr.get_metrics(verbose=True), want)
