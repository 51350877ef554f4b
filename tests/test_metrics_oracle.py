"""oracle/metrics_oracle.py reproduces the fixtures made by executing the reference's trackers
(oracle/make_golden_metrics.py): confusion matrices as integers, metrics as float64, full-resolution predictions
element for element.  CPU only."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import metrics_oracle as MO

K = 6


def fixture(name):
    z = np.load(os.path.join(GOLDEN, f"metrics_{name}.npz"), allow_pickle=False)
    return {k: z[k] for k in z.files}, json.loads(str(z["metrics"]))


def check_segmentation_keys(m, stage, cm):
    acc, macc, miou, iou = MO.metrics(cm)
    assert m[f"{stage}_acc"] == 100 * acc and m[f"{stage}_macc"] == 100 * macc and m[f"{stage}_miou"] == 100 * miou
    assert m[f"{stage}_miou_per_class"] == {str(i): "{:.2f}".format(100 * v) for i, v in enumerate(iou)}


def test_segmentation():
    z, m = fixture("segmentation")
    cm = MO.segmentation(z["scores"], z["labels"], K)
    assert (cm == z["cm"]).all()
    check_segmentation_keys(m, "val", cm)


def test_s3dis():
    z, m = fixture("s3dis")
    assert (MO.segmentation(z["scores"], z["labels"], K) == z["cm"]).all()
    vcm, pred, fcm = MO.s3dis(z["pos"], z["y"], K, list(z["ids"]), list(z["scores"]))
    assert (pred == z["full_pred"]).all() and (fcm == z["full_cm"]).all()
    _, _, vmiou, viou = MO.metrics(vcm)
    assert m["test_vote_miou"] == 100 * vmiou
    assert m["test_vote_iou"] == {f"c{k}": 100 * v for k, v in enumerate(viou)}
    _, _, fmiou, fiou = MO.metrics(fcm)
    assert m["test_full_vote_miou"] == 100 * fmiou
    assert m["test_iou"] == {f"c{k}": v for k, v in enumerate(MO.metrics(z["cm"])[3])}
    check_segmentation_keys(m, "test", z["cm"])


def test_scannet():
    z, m = fixture("scannet")
    raws = {s: (z[f"pos{s}"], z[f"y{s}"]) for s in (0, 1)}
    samples = []
    b = 0
    while f"b{b}/id_scan" in z:
        for i, s in enumerate(z[f"b{b}/id_scan"]):
            sel = z[f"b{b}/batch"] == i
            samples.append((int(s), z[f"b{b}/origin_id"][sel], z[f"b{b}/scores"][sel]))
        b += 1
    preds, fcm = MO.scannet(raws, K, samples)
    for s in (0, 1):
        assert (preds[s] == z[f"full_pred{s}"]).all()
    assert (fcm == z["full_cm"]).all()
    acc, macc, miou, _ = MO.metrics(fcm)
    assert m["val_full_acc"] == 100 * acc and m["val_full_macc"] == 100 * macc and m["val_full_miou"] == 100 * miou


def test_kitti360():
    z, m = fixture("kitti360")
    windows = [(z[f"pos{w}"], z[f"y{w}"]) for w in range(3)]
    samples = [(int(w), z[f"s{i}/ids"], z[f"s{i}/scores"]) for i, w in enumerate(z["order"])]
    vcm, fcm = MO.kitti360(windows, K, samples)
    assert (vcm == z["vote_cm"]).all() and (fcm == z["full_cm"]).all()
    assert m["val_vote_miou"] == 100 * MO.metrics(vcm)[2]
    assert m["val_full_miou"] == 100 * MO.metrics(fcm)[2]


def test_knn_interpolate_zero_distance_rounding():
    """At d = 0, w = 1e16 and (x w) / w is computed as such: the stand-in does not shortcut to x."""
    x = torch.tensor([[3.0000002, 3.0]])
    y = MO.knn_interpolate(x, torch.zeros(1, 3), torch.zeros(1, 3))
    w = torch.tensor(1e16)
    assert torch.equal(y, (x * w) / w)


@pytest.mark.parametrize("cls", ["APIModel", "No3DLogitFusion"])
def test_models_expose_the_tracker_interface(cls):
    from deepviewagg_b200.models.multimodal import no3d, sparseconv3d
    mod = sparseconv3d if cls == "APIModel" else no3d
    model = getattr(mod, cls).__new__(getattr(mod, cls))
    torch.nn.Module.__init__(model)
    model._modalities = ["image"]
    data = type("D", (), {"y": torch.tensor([1, 2]), "batch": torch.tensor([0, 0])})()
    model.set_input(data)
    model.output = torch.zeros(2, K)
    assert model.get_input() is data and model.get_output() is model.output
    assert torch.equal(model.get_labels(), data.y)
    assert model.is_multimodal
    model._modalities = []
    assert not model.is_multimodal
