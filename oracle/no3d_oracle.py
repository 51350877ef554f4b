"""numpy restatement of the No3D models (TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py; never
imported by the product path), pinned on tests/golden/no3d_*.npz by tests/test_no3d_oracle.py.

Restates, for the fixtures' configuration (one MultimodalBlockDown, one pixel per view, atomic max
pool, view mean pool, residual fusion of x_3d = None), models/segmentation/multimodal/no3d.py:73-157
and applications/multimodal/no3d.py:79-130, plus the brute-force nearest-neighbour search of a
query set among a search set (KeOps `argmin` of no3d.py:116-120; `knn_query_bruteforce`).
"""
import numpy as np


def knn_query_bruteforce(query, search, k, block=512):
    """k nearest search points of every query point; squared distances (dx*dx + dy*dy) + dz*dz in
    float32, ascending (dist, search index).  Returns (neighbors [M,k] int64, dist2 [M,k] float32)."""
    q_all = np.asarray(query, dtype=np.float32)
    p = np.asarray(search, dtype=np.float32)
    m = q_all.shape[0]
    nbr = np.empty((m, k), dtype=np.int64)
    d2o = np.empty((m, k), dtype=np.float32)
    for s in range(0, m, block):
        q = q_all[s:s + block]
        dx = q[:, None, 0] - p[None, :, 0]
        dy = q[:, None, 1] - p[None, :, 1]
        dz = q[:, None, 2] - p[None, :, 2]
        d2 = (dx * dx + dy * dy) + dz * dz
        idx = np.argsort(d2, axis=1, kind="stable")[:, :k]
        nbr[s:s + block] = idx
        d2o[s:s + block] = np.take_along_axis(d2, idx, axis=1)
    return nbr, d2o


def log_softmax(x):
    x = np.asarray(x, dtype=np.float64)
    m = x.max(axis=1, keepdims=True)
    return x - m - np.log(np.exp(x - m).sum(axis=1, keepdims=True))


def nll_mean(logp, target, ignore_index=-1):
    keep = target != ignore_index
    if not keep.any():
        return float("nan")
    return float(-logp[keep, target[keep]].mean())


def _mlp(x, sd, prefix, training, eps=1e-5):
    """MLP([C, C'], ReLU, bias=False) of base_modules.py:38-48 (one layer)."""
    z = x @ sd[prefix + "0.0.weight"].astype(np.float64).T
    if training:
        mean, var = z.mean(0), z.var(0)
    else:
        mean = sd[prefix + "0.1.batch_norm.running_mean"].astype(np.float64)
        var = sd[prefix + "0.1.batch_norm.running_var"].astype(np.float64)
    z = (z - mean) / np.sqrt(var + eps) * sd[prefix + "0.1.batch_norm.weight"] + sd[prefix + "0.1.batch_norm.bias"]
    return np.maximum(z, 0)


def no3d_forward(cls_name, training, pos, labels, settings, maps, sd, x3d=None):
    """settings: per setting dict(pid, iid, pix); maps: per setting [n_img, C, H, W]; sd: the model's
    state dict (numpy).  Returns (output [N, K] log-probs, loss, labels after the in-place masking)."""
    n = pos.shape[0]
    labels = labels.copy()
    has_head = "Feature" in cls_name
    view_loss = cls_name.startswith("No3DImage")
    if settings:
        # atomic max pool of one pixel per view = the pixel's feature; view mean pool per point
        pid = np.concatenate([s["pid"] for s in settings])
        feats = np.concatenate([m[s["iid"], :, s["pix"][:, 1], s["pix"][:, 0]] for s, m in zip(settings, maps)])
        feats = feats.astype(np.float64)
        order = np.argsort(pid, kind="stable")
        pid, feats = pid[order], feats[order]
        counts = np.bincount(pid, minlength=n)
        x = np.zeros((n, feats.shape[1]))
        np.add.at(x, pid, feats)
        seen = counts > 0
        x[seen] /= counts[seen, None]
    else:
        x, seen = np.asarray(x3d, dtype=np.float64), np.zeros(n, dtype=bool)
        pid, feats = np.zeros(0, dtype=np.int64), None
    if "backbone.mlp.0.0.weight" in sd:
        x = _mlp(x, sd, "backbone.mlp.", training)
        if feats is not None:
            feats = _mlp(feats, sd, "backbone.mlp.", training)
    if has_head:
        w, b = sd["head.0.weight"].astype(np.float64), sd["head.0.bias"].astype(np.float64)
        head = lambda t: t @ w.T + b  # noqa: E731
    else:
        head = lambda t: t  # noqa: E731
    out = log_softmax(head(x))
    if not training and seen.any():
        unseen = np.nonzero(~seen)[0]
        if unseen.size:
            seen_idx = np.nonzero(seen)[0]
            nn_idx, _ = knn_query_bruteforce(pos[unseen], pos[seen_idx], 1)
            out[unseen] = out[seen_idx[nn_idx[:, 0]]]
    else:
        labels[~seen] = -1
    if view_loss:
        loss = nll_mean(log_softmax(head(feats)), labels[pid])
    else:
        loss = nll_mean(out, labels)
    return out, loss, labels
