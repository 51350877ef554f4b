"""Generate the segmentation-metric fixtures by EXECUTING THE REFERENCE (oracle; test infrastructure).

Run in the build container only (needs the reference checkout, see oracle/ref_loader.py):
    python -m oracle.make_golden_metrics
writes tests/golden/metrics_{segmentation,s3dis,scannet,kitti360}.npz.

The reference's metrics/confusion_matrix.py, base_tracker.py, segmentation_tracker.py, s3dis_tracker.py,
scannet_segmentation_tracker.py and kitti360_tracker.py are loaded by path and run unchanged, with stand-ins for
their parents and for what a trainer provides: torchnet / wandb / tensorboard (loss meters and loggers, unused
here), IGNORE_LABEL = -1, SaveOriginalPosId.KEY = 'origin_id', a model exposing get_output / get_labels /
get_input / get_current_losses, duck-typed datasets, and read_kitti360_window returning the window of the fixture.
torch_geometric's knn_interpolate is bound to oracle/metrics_oracle.knn_interpolate, which is RESTATED, NOT
EXECUTED (k = 1, exhaustive search, ties to the lower index; the interpolation arithmetic in torch_geometric's
order).  Scenarios: overlapping samples over several voting runs, ignored labels, an absent class, exact score
ties, NaN rows (in the per-batch tracker, whose argmax is numpy's), regions far from every voted point, a
multi-window KITTI-360 run with window switches, and ScanNet batches of two scans.

Each fixture holds the inputs, the reference's confusion matrices, its get_metrics(verbose=True) dict as JSON
(`metrics`) and, where the reference keeps them or passes them through knn_interpolate, the full-resolution
predictions."""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import metrics_oracle as MO  # noqa: E402
from oracle import ref_loader  # noqa: E402

K = 6                     # class 5 never appears in any label: an absent class
OUT = os.path.join(ROOT, "tests", "golden")


def load_reference_metrics():
    st = ref_loader._stub
    for pkg in ["torch_points3d", "torch_points3d.metrics", "torch_points3d.datasets",
                "torch_points3d.datasets.segmentation", "torch_points3d.core", "torch_points3d.core.data_transform",
                "torch_points3d.models", "torch_geometric", "torch_geometric.nn", "torch_geometric.nn.unpool",
                "torch_geometric.data", "torchnet", "wandb", "torch.utils.tensorboard"]:
        st(pkg)
    tn = sys.modules["torchnet"]
    tn.meter = types.SimpleNamespace(AverageValueMeter=object)
    sys.modules["torch.utils.tensorboard"].SummaryWriter = object
    sys.modules["torch_points3d.datasets.segmentation"].IGNORE_LABEL = -1
    sys.modules["torch_points3d.core.data_transform"].SaveOriginalPosId = type("SaveOriginalPosId", (),
                                                                                {"KEY": "origin_id"})
    sys.modules["torch_points3d.models"].model_interface = types.SimpleNamespace(TrackerInterface=object)
    sys.modules["torch_geometric.nn.unpool"].knn_interpolate = MO.knn_interpolate
    sys.modules["torch_geometric.data"].Batch = type("Batch", (), {})
    st("torch_points3d.metrics.meters").APMeter = object
    st("torch_points3d.datasets.batch").SimpleBatch = type("SimpleBatch", (), {})
    st("torch_points3d.datasets.segmentation.kitti360").read_kitti360_window = _read_window
    st("torch_points3d.datasets.segmentation.kitti360_config").TRAINID2ID = np.arange(K)
    ns = types.SimpleNamespace()
    for name in ("confusion_matrix", "base_tracker", "segmentation_tracker", "s3dis_tracker",
                 "scannet_segmentation_tracker", "kitti360_tracker"):
        setattr(ns, name, ref_loader._load(f"torch_points3d.metrics.{name}", f"torch_points3d/metrics/{name}.py"))
    return ns


_WINDOWS = {}


def _read_window(path, xyz=True, rgb=False, semantic=True, instance=False, remap=True):
    pos, y = _WINDOWS[path]
    return types.SimpleNamespace(pos=torch.from_numpy(pos), y=torch.from_numpy(y))


class Model:
    is_multimodal = False
    conv_type = "SPARSE"
    device = "cpu"

    def __init__(self, out, y, inp=None):
        self.out, self.y, self.inp = out, y, inp

    def get_output(self):
        return self.out

    def get_labels(self):
        return self.y

    def get_input(self):
        return self.inp

    def get_current_losses(self):
        return {}


class Dataset:
    def __init__(self, **kw):
        self.num_classes = K
        self.INV_OBJECT_LABEL = {i: f"c{i}" for i in range(K)}
        self.__dict__.update(kw)

    def has_labels(self, stage):
        return True


class Sample(dict):
    """Attribute and item access, as torch_geometric's Data gives."""
    __getattr__ = dict.__getitem__

    def __setattr__(self, k, v):
        self[k] = v


class IdScans(list):
    """id_scan of a batch: .dim() / .squeeze() as a tensor, iterated as ints (the tracker keys its dicts on them)."""

    def dim(self):
        return 1

    def squeeze(self):
        return self


class Area:
    def __init__(self, pos, y):
        self.pos, self.y = torch.from_numpy(pos), torch.from_numpy(y)

    def clone(self):
        return Area(self.pos.numpy().copy(), self.y.numpy().copy())

    def to(self, device):
        return self


def scores(rng, n, ties=True, nan=False):
    s = rng.standard_normal((n, K)).astype(np.float32)
    s[:, 5] -= 3.0                                      # the absent class is rarely predicted
    if ties:
        r = rng.choice(n, n // 10, replace=False)
        s[r, 2] = s[r, 1] = np.maximum(s[r, 1], s[r, 2]) + 1.0      # exact ties between classes 1 and 2
    if nan:
        r = rng.choice(n, n // 25, replace=False)
        s[r, rng.integers(0, K, r.size)] = np.nan
    return s


def cloud(rng, n, far_share=0.15):
    pos = (rng.random((n, 3)) * [10.0, 10.0, 2.0]).astype(np.float32)
    pos = np.round(pos * 50) / 50                        # a 2 cm lattice: exact distance ties
    far = rng.random(n) < far_share
    pos[far, 0] += 30.0                                  # a region far from the sampled part
    return pos.astype(np.float32), far


def labels(rng, n, ignore_share=0.0):
    y = rng.integers(0, K - 1, n).astype(np.int64)
    y[rng.random(n) < ignore_share] = -1
    return y


def save(name, **arrays):
    path = os.path.join(OUT, f"metrics_{name}.npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path)


def js(metrics):
    def conv(v):
        if isinstance(v, dict):
            return {str(k): conv(x) for k, x in v.items()}
        return v if isinstance(v, str) else float(v)
    return json.dumps({k: conv(v) for k, v in metrics.items()})


def gen_segmentation(R, rng):
    B, n = 6, 500
    S = np.stack([scores(rng, n, nan=True) for _ in range(B)])
    Y = np.stack([labels(rng, n, 0.1) for _ in range(B)])
    Y[3] = -1                                            # a batch whose labels are all ignored
    tr = R.segmentation_tracker.SegmentationTracker(Dataset(), stage="val")
    for s, y in zip(S, Y):
        tr.track(Model(torch.from_numpy(s), torch.from_numpy(y)))
    save("segmentation", scores=S, labels=Y, cm=tr.confusion_matrix, metrics=js(tr.get_metrics(verbose=True)))


def gen_s3dis(R, rng):
    N, B, n = 3000, 10, 400
    pos, far = cloud(rng, N)
    y = labels(rng, N)
    near = np.flatnonzero(~far)
    ids = np.stack([rng.choice(near, n, replace=False) for _ in range(B)])   # overlapping spheres, several runs
    S = np.stack([scores(rng, n) for _ in range(B)])
    L = y[ids].copy()
    L[:, :40] = -1
    calls = []
    real = MO.knn_interpolate

    def recording(*a, **kw):
        out = real(*a, **kw)
        calls.append(out)
        return out
    R.s3dis_tracker.knn_interpolate = recording
    tr = R.s3dis_tracker.S3DISTracker(Dataset(test_data=Area(pos, y)), stage="test")
    for i, s, lab in zip(ids, S, L):
        tr.track(Model(torch.from_numpy(s), torch.from_numpy(lab), {"origin_id": torch.from_numpy(i)}), full_res=True)
    tr.finalise(full_res=True, vote_miou=True)
    R.s3dis_tracker.knn_interpolate = real
    save("s3dis", pos=pos, y=y, ids=ids, scores=S, labels=L, cm=tr.confusion_matrix,
         full_cm=tr.full_confusion_matrix.confusion_matrix, full_pred=MO.argmax(calls[0].numpy()),
         metrics=js(tr.get_metrics(verbose=True)))


def gen_scannet(R, rng):
    sizes = (1500, 1200)
    raws = {}
    for sid, n in enumerate(sizes):
        pos, _ = cloud(rng, n)
        raws[sid] = (pos, labels(rng, n, 0.1))
    ds = Dataset()
    ds.get_raw_data = lambda stage, i, remap_labels=True: types.SimpleNamespace(
        pos=torch.from_numpy(raws[i][0]), y=torch.from_numpy(raws[i][1]))
    tr = R.scannet_segmentation_tracker.ScannetSegmentationTracker(ds, stage="val")
    batches = []
    for b in range(5):
        scans = [b % 2, (b + 1) % 2] if b < 4 else [1, 1]
        per = [rng.choice(int(sizes[s] * 0.8), 300, replace=False) for s in scans]   # the last 20 % unvoted
        origin = np.concatenate(per)
        batch = np.repeat(np.arange(len(scans)), 300)
        s = scores(rng, origin.size)
        lab = np.concatenate([raws[sc][1][p] for sc, p in zip(scans, per)])
        data = Sample(id_scan=IdScans(scans), batch=torch.from_numpy(batch), origin_id=torch.from_numpy(origin))
        tr.track(Model(torch.from_numpy(s), torch.from_numpy(lab)), full_res=True, data=data)
        batches.append((np.array(scans), origin, batch, s, lab))
    tr.finalise(full_res=True)
    arrays = {"metrics": js(tr.get_metrics(verbose=True)), "cm": tr.confusion_matrix,
              "full_cm": tr._full_confusion_matrix.confusion_matrix}
    for sid, (pos, y) in raws.items():
        arrays[f"pos{sid}"], arrays[f"y{sid}"] = pos, y
        arrays[f"full_pred{sid}"] = tr._full_preds[sid].numpy()
    for b, (scans, origin, batch, s, lab) in enumerate(batches):
        arrays.update({f"b{b}/id_scan": scans, f"b{b}/origin_id": origin, f"b{b}/batch": batch, f"b{b}/scores": s,
                       f"b{b}/labels": lab})
    save("scannet", **arrays)


def gen_kitti360(R, rng):
    sizes = (1500, 1000, 1200)
    windows = [f"seq_0/w{i}" for i in range(len(sizes))]
    wins = []
    for w, n in enumerate(sizes):
        pos, _ = cloud(rng, n, far_share=0.25)
        y = labels(rng, n, 0.1)
        wins.append((pos, y))
        _WINDOWS[f"/raw/{windows[w]}.ply"] = (pos, y)
    stage = types.SimpleNamespace(windows=windows, raw_dir="/raw", raw_file_names_3d=[w + ".ply" for w in windows],
                                  window_raw_sizes=list(sizes))
    ds = Dataset(submission_dir="/nonexistent")
    ds.get_dataset = lambda stage_name: stage
    tr = R.kitti360_tracker.KITTI360Tracker(ds, stage="val")
    order = [0, 0, 1, 0, 2, 2, 1, 0, 2]                  # window switches, returns to earlier windows
    samples = []
    for w in order:
        ids = rng.choice(int(sizes[w] * 0.7), 250, replace=False)
        s = scores(rng, 250)
        lab = wins[w][1][ids]
        data = Sample(idx_window=w, origin_id=torch.from_numpy(ids))
        tr.track(Model(torch.from_numpy(s), torch.from_numpy(lab)), data=data)
        samples.append((w, ids, s, lab))
    tr.finalise(full_res=True)
    arrays = {"metrics": js(tr.get_metrics(verbose=True)), "cm": tr.confusion_matrix,
              "vote_cm": tr._vote_confusion_matrix.confusion_matrix,
              "full_cm": tr._full_confusion_matrix.confusion_matrix, "order": np.array(order)}
    for w, (pos, y) in enumerate(wins):
        arrays[f"pos{w}"], arrays[f"y{w}"] = pos, y
    for i, (w, ids, s, lab) in enumerate(samples):
        arrays.update({f"s{i}/ids": ids, f"s{i}/scores": s, f"s{i}/labels": lab})
    save("kitti360", **arrays)


def main():
    R = load_reference_metrics()
    rng = np.random.default_rng(20261016)
    gen_segmentation(R, rng)
    gen_s3dis(R, rng)
    gen_scannet(R, rng)
    gen_kitti360(R, rng)


if __name__ == "__main__":
    main()
