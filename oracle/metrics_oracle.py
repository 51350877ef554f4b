"""numpy / torch-CPU restatement of the reference's segmentation evaluation (oracle; test infrastructure).

  * confusion(gt, pred, K): metrics/confusion_matrix.py count_predicted_batch (np.bincount of K * gt + pred);
  * metrics(cm): the float64 formulas of confusion_matrix.py (acc, macc, mIoU, per-class IoU);
  * knn_interpolate(x, pos_x, pos_y, k=1): torch_geometric's k = 1 knn_interpolate RESTATED, NOT EXECUTED
    (torch_geometric / torch_cluster are not installed): the nearest point of pos_x by exhaustive search,
    d2 = (dx dx + dy dy) + dz dz in fp32, ties to the lower index (torch_cluster's tie order is undocumented),
    then diff = pos_x[idx] - pos_y, w = 1 / clamp(d2, 1e-16), y = (x[idx] w) / w, each step an fp32 op;
  * s3dis / scannet / kitti360 / segmentation: the trackers' bookkeeping on the fixtures' inputs.
oracle/make_golden_metrics.py binds knn_interpolate in place of torch_geometric's when it executes the reference's
trackers; tests/test_metrics_oracle.py checks that these functions reproduce the fixtures."""
import numpy as np
import torch


def confusion(gt, pred, K):
    return np.bincount(K * np.asarray(gt).astype(int) + np.asarray(pred), minlength=K * K).reshape(K, K)


def metrics(cm):
    cm = np.asarray(cm)
    tp = np.diagonal(cm)
    union = np.sum(cm, axis=0) + np.sum(cm, axis=1) - tp
    iou = 1e-8 + tp / (union + 1e-8)
    ex = union > 1e-3
    miou = np.sum(iou[ex]) / np.sum(ex) if np.sum(ex) else 0
    total = int(cm.sum())
    acc = float(int(np.trace(cm))) / (total if total else 1)
    re, present = 0, 0
    for i in range(cm.shape[0]):
        t = np.sum(cm[i, :])
        if t:
            present += 1
            re = re + cm[i][i] / max(1, t)
    return acc, (re / present if present else 0), miou, iou


def nearest(pos_x, pos_y, chunk=2048):
    """Index into pos_x of the nearest point of every pos_y row, fp32 (dx dx + dy dy) + dz dz, lowest index on ties."""
    px, py = torch.as_tensor(pos_x, dtype=torch.float32), torch.as_tensor(pos_y, dtype=torch.float32)
    out = torch.empty(py.shape[0], dtype=torch.int64)
    ar = torch.arange(px.shape[0])
    for s in range(0, py.shape[0], chunk):
        d = px[None, :, :] - py[s:s + chunk, None, :]
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        m = d2.min(1, keepdim=True).values
        out[s:s + chunk] = torch.where(d2 == m, ar, px.shape[0]).min(1).values
    return out


def knn_interpolate(x, pos_x, pos_y, batch_x=None, batch_y=None, k=1, num_workers=1):
    assert k == 1 and batch_x is None and batch_y is None
    x, pos_x, pos_y = torch.as_tensor(x).float(), torch.as_tensor(pos_x).float(), torch.as_tensor(pos_y).float()
    idx = nearest(pos_x, pos_y)
    diff = pos_x[idx] - pos_y
    d2 = ((diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1]) + diff[:, 2] * diff[:, 2])[:, None]
    w = 1.0 / torch.clamp(d2, min=1e-16)
    return (x[idx] * w) / w


def argmax(t):
    return np.argmax(np.asarray(t, dtype=np.float32), 1)


def segmentation(scores, labels, K, ignore=-1):
    """Per-batch confusion of SegmentationTracker over batches of scores [B, n, K] and labels [B, n]."""
    cm = np.zeros((K, K), dtype=np.int64)
    for s, y in zip(scores, labels):
        m = y != ignore
        if m.any():
            cm += confusion(y[m], argmax(s[m]), K)
    return cm


def vote(N, K, ids_list, out_list):
    """votes[ids] += out; counts[ids] += 1 over the batches (ids unique within a batch)."""
    votes, counts = torch.zeros(N, K), torch.zeros(N, dtype=torch.int32)
    for ids, out in zip(ids_list, out_list):
        ids = torch.as_tensor(ids)
        votes[ids] += torch.as_tensor(out)
        counts[ids] += 1
    return votes, counts


def s3dis(pos, y, K, ids_list, out_list):
    """(vote confusion, full-resolution predictions, full confusion) of S3DISTracker.finalise(full_res=True)."""
    votes, counts = vote(pos.shape[0], K, ids_list, out_list)
    has = (counts > 0).numpy()
    vcm = confusion(y[has], argmax(votes.numpy()[has]), K)
    pred = argmax(knn_interpolate(votes[torch.from_numpy(has)], pos[has], pos).numpy())
    return vcm, pred, confusion(y, pred, K)


def scannet(raws, K, samples, ignore=-1):
    """Full-resolution predictions per scan and the full confusion of ScannetSegmentationTracker; samples are
    (id_scan, origin ids, outputs)."""
    acc = {}
    for id_scan, ids, out in samples:
        acc.setdefault(id_scan, ([], []))
        acc[id_scan][0].append(ids)
        acc[id_scan][1].append(out)
    preds, cm = {}, np.zeros((K, K), dtype=np.int64)
    for id_scan, (ids_list, out_list) in acc.items():
        pos, y = raws[id_scan]
        votes, counts = vote(pos.shape[0], K, ids_list, out_list)
        has = counts > 0
        votes[has] /= counts[has].unsqueeze(-1)
        pred = argmax(knn_interpolate(votes[has], pos[has.numpy()], pos).numpy())
        preds[id_scan] = pred
        m = y != ignore
        cm += confusion(y[m], pred[m], K)
    return preds, cm


def kitti360(windows, K, samples, ignore=-1):
    """(vote confusion, full confusion) of KITTI360Tracker.finalise(full_res=True) over windows (pos, y); samples
    are (idx_window, origin ids, outputs)."""
    vcm, fcm = np.zeros((K, K), dtype=np.int64), np.zeros((K, K), dtype=np.int64)
    for w, (pos, y) in enumerate(windows):
        ids_list = [s[1] for s in samples if s[0] == w]
        out_list = [s[2] for s in samples if s[0] == w]
        votes, counts = vote(pos.shape[0], K, ids_list, out_list)
        has = (counts > 0).numpy()
        pred = argmax(votes.numpy()[has])
        gt = y[has]
        m = gt != ignore
        vcm += confusion(gt[m], pred[m], K)
        full = argmax(votes.numpy())
        full[~has] = argmax(knn_interpolate(votes[torch.from_numpy(has)], pos[has], pos[~has]).numpy())
        m = y != ignore
        fcm += confusion(y[m], full[m], K)
    return vcm, fcm
