"""float64 numpy restatement of the Lovász-softmax loss (TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py;
never imported by the product path), pinned on tests/golden/lovasz_*.npz by tests/test_sparseconv3d_oracle.py.

Restates lovasz_softmax_flat(*flatten_probas(probas, labels, ignore), classes) and lovasz_grad of
metrics/lovasz_loss.py:18-30, 155-230 for [P, K] inputs, and its gradient with respect to probas.  The sort is
a stable descending argsort: tied errors keep point order (the reference's CPU torch.sort is unstable, so on
tied inputs only the loss is comparable).  With no valid point, or no kept class, the loss is 0 and the gradient
0 (the reference returns `probas * 0.` of shape [0, K], and mean([]) = 0).
"""
import numpy as np


def lovasz_grad(fg_sorted):
    """Jaccard differences of a sorted fg vector (lovasz_loss.py:18-30)."""
    fg = np.asarray(fg_sorted, dtype=np.float64)
    gts = fg.sum()
    intersection = gts - np.cumsum(fg)
    union = gts + np.cumsum(1.0 - fg)
    jaccard = 1.0 - intersection / union
    if fg.size > 1:
        jaccard[1:] = jaccard[1:] - jaccard[:-1]
    return jaccard


def lovasz_softmax(probas, labels, classes="present", ignore=-1):
    """(loss, grad [P, K], per-class losses {c: loss_c}) in float64."""
    probas = np.asarray(probas, dtype=np.float64)
    labels = np.asarray(labels)
    P, K = probas.shape
    grad = np.zeros_like(probas)
    valid = labels != ignore
    vp, vl = probas[valid], labels[valid]
    vidx = np.nonzero(valid)[0]
    if vp.shape[0] == 0:
        return 0.0, grad, {}
    todo = list(range(K)) if classes in ("all", "present") else [int(c) for c in classes]
    losses, per_class, grads = [], {}, []
    for c in todo:
        fg = (vl == c).astype(np.float64)
        if classes == "present" and fg.sum() == 0:
            continue
        d = fg - vp[:, c]
        err = np.abs(d)
        perm = np.argsort(-err, kind="stable")
        g = lovasz_grad(fg[perm])
        loss_c = float(np.dot(err[perm], g))
        losses.append(loss_c)
        per_class[c] = loss_c
        gc = np.zeros(vp.shape[0])
        gc[perm] = g
        grads.append((c, -np.sign(d) * gc))
    if not losses:
        return 0.0, grad, per_class
    n = len(losses)
    for c, gc in grads:
        grad[vidx, c] += gc / n
    return float(sum(losses) / n), grad, per_class


def sorted_blocks(probas, labels, c, ignore=-1):
    """Tied blocks of class c: a list of arrays of point indices whose errors |fg - p| are equal (valid points)."""
    probas = np.asarray(probas, dtype=np.float64)
    labels = np.asarray(labels)
    idx = np.nonzero(labels != ignore)[0]
    err = np.abs((labels[idx] == c).astype(np.float64) - probas[idx, c])
    order = np.argsort(-err, kind="stable")
    e = err[order]
    cuts = np.nonzero(np.diff(e) != 0)[0] + 1
    return [idx[order[s]] for s in np.split(np.arange(e.size), cuts)]
