"""Segmentation evaluation on the GPU (ops.confusion_update / vote / full_res_predict and deepviewagg_b200.metrics)
against numpy and torch restatements of the reference's trackers.  Every result is an integer, an argmax or an
exact fp32 sequence, so everything is compared for equality."""
import types

import numpy as np
import pytest
import torch

from deepviewagg_b200 import ops
from deepviewagg_b200.metrics import ConfusionMatrix, S3DISTracker, SegmentationTracker

pytestmark = pytest.mark.gpu
DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}


def np_confusion(gt, pred, K):
    """metrics/confusion_matrix.py count_predicted_batch: bincount(K * gt + pred)."""
    return np.bincount(K * np.asarray(gt).astype(int) + np.asarray(pred), minlength=K * K).reshape(K, K)


def np_argmax(scores):
    return np.argmax(scores.float().cpu().numpy(), 1)


# ---------------------------------------------------------------------------------------------------------------
# the per-batch update
# ---------------------------------------------------------------------------------------------------------------
def scores_scenario(dt, n=383_000, K=13, seed=0):
    """The S3DIS step shape: 10 % ignored labels, the confusion equals bincount of torch's argmax."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    scores = torch.randn(n, K, generator=g, device="cuda").to(DTYPES[dt])
    labels = torch.randint(0, K, (n,), generator=g, device="cuda")
    labels[torch.rand(n, generator=g, device="cuda") < 0.1] = -1
    cm = torch.zeros(K, K, dtype=torch.int64, device="cuda")
    status = ops.confusion_update(cm, scores, labels, ignore_label=-1)
    keep = labels != -1
    ref = torch.bincount(K * labels[keep] + scores[keep].argmax(1), minlength=K * K).view(K, K)
    assert torch.equal(cm, ref)
    assert int(status.item()) == 0
    # counts: rows with count 0 are skipped
    counts = (torch.rand(n, generator=g, device="cuda") < 0.5).int()
    cm2 = torch.zeros_like(cm)
    ops.confusion_update(cm2, scores, labels, ignore_label=-1, counts=counts)
    keep2 = keep & (counts > 0)
    ref2 = torch.bincount(K * labels[keep2] + scores[keep2].argmax(1), minlength=K * K).view(K, K)
    assert torch.equal(cm2, ref2)
    return cm


@pytest.mark.parametrize("dt", list(DTYPES))
def test_confusion_at_the_s3dis_step_shape(dt):
    scores_scenario(dt)


def pred_scenario(n=100_000, K=20):
    g = torch.Generator(device="cuda").manual_seed(1)
    pred = torch.randint(0, K, (n,), generator=g, device="cuda")
    labels = torch.randint(0, K, (n,), generator=g, device="cuda")
    cm = torch.zeros(K, K, dtype=torch.int64, device="cuda")
    status = ops.confusion_update(cm, pred, labels)
    assert torch.equal(cm.cpu(), torch.from_numpy(np_confusion(labels.cpu().numpy(), pred.cpu().numpy(), K)))
    assert int(status.item()) == 0


def test_confusion_from_predictions():
    pred_scenario()


def test_numpy_argmax_rule_ties_and_nan():
    K = 7
    rows = torch.tensor([[1, 3, 3, 0, 0, 0, 0],           # tie: first index
                         [2, 2, 2, 2, 2, 2, 2],           # all equal: 0
                         [0, float("nan"), 5, float("nan"), 0, 0, 0],   # first NaN wins
                         [float("nan"), 9, 9, 9, 9, 9, 9],
                         [-float("inf"), -float("inf"), -5, 0, float("inf"), float("inf"), 0]])
    labels = torch.arange(5) % K
    want = np.argmax(rows.numpy(), 1)
    assert list(want) == [1, 0, 1, 0, 4]
    for dt in DTYPES.values():
        cm = torch.zeros(K, K, dtype=torch.int64, device="cuda")
        ops.confusion_update(cm, rows.to(dt).cuda(), labels.cuda())
        assert torch.equal(cm.cpu(), torch.from_numpy(np_confusion(labels.numpy(), want, K)))


def test_64_classes_work_and_65_raise():
    n = 50_000
    g = torch.Generator(device="cuda").manual_seed(2)
    scores = torch.randn(n, 64, generator=g, device="cuda")
    labels = torch.randint(0, 64, (n,), generator=g, device="cuda")
    cm = torch.zeros(64, 64, dtype=torch.int64, device="cuda")
    ops.confusion_update(cm, scores, labels)
    assert torch.equal(cm, torch.bincount(64 * labels + scores.argmax(1), minlength=64 * 64).view(64, 64))
    with pytest.raises(ValueError, match="65 classes"):
        ops.confusion_update(torch.zeros(65, 65, dtype=torch.int64, device="cuda"), torch.randn(4, 65, device="cuda"),
                             torch.zeros(4, dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError, match="65 classes"):
        ops.vote(torch.zeros(4, 65, device="cuda"), torch.zeros(4, dtype=torch.int32, device="cuda"),
                 torch.full((4,), -1, dtype=torch.int32, device="cuda"), torch.zeros(2, dtype=torch.int64, device="cuda"),
                 torch.zeros(2, 65, device="cuda"))
    with pytest.raises(ValueError, match="65 classes"):
        ops.full_res_predict(torch.zeros(4, 65, device="cuda"), torch.ones(4, dtype=torch.int32, device="cuda"),
                             torch.zeros(4, 3, device="cuda"))


def test_out_of_range_labels_raise_at_the_first_read():
    K = 5
    c = ConfusionMatrix(K)
    scores = torch.randn(10, K, device="cuda")
    c.count_scores_batch(torch.tensor([0, 1, 2, 3, 4, 5, 0, 1, 2, -1], device="cuda"), scores, ignore_label=-1)
    with pytest.raises(ValueError, match="label outside"):
        c.get_average_intersection_union()
    c = ConfusionMatrix(K)
    c.count_predicted_batch(torch.tensor([0, 1], device="cuda"), torch.tensor([0, 7], device="cuda"))
    with pytest.raises(ValueError, match="prediction outside"):
        c.get_overall_accuracy()
    # numpy / CPU inputs are copied once and counted the same way
    c = ConfusionMatrix(K)
    c.count_predicted_batch(np.array([0, 1, 1, 4]), torch.tensor([0, 1, 2, 4]))
    assert (c.confusion_matrix == np_confusion([0, 1, 1, 4], [0, 1, 2, 4], K)).all()


# ---------------------------------------------------------------------------------------------------------------
# votes
# ---------------------------------------------------------------------------------------------------------------
def vote_scenario(dt, N=200_000, n=60_000, K=13):
    g = torch.Generator(device="cuda").manual_seed(3)
    votes = torch.randn(N, K, generator=g, device="cuda")
    counts = torch.randint(0, 4, (N,), generator=g, device="cuda", dtype=torch.int32)
    stamp = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = torch.randn(n, K, generator=g, device="cuda").to(DTYPES[dt])
    # unique ids: bit-equal to index_put_
    ids = torch.randperm(N, generator=g, device="cuda")[:n]
    ref_v, ref_c = votes.clone(), counts.clone()
    ref_v[ids] += out
    ref_c[ids] += 1
    status = ops.vote(votes, counts, stamp, ids, out)
    assert torch.equal(votes.view(torch.int32), ref_v.view(torch.int32))
    assert torch.equal(counts, ref_c)
    assert bool((stamp == -1).all()) and int(status.item()) == 0
    # duplicated ids: the last occurrence wins
    dup = torch.randint(0, N // 50, (n,), generator=g, device="cuda")
    ref_v, ref_c = votes.clone(), counts.clone()
    last = {}
    for j, i in enumerate(dup.tolist()):
        last[i] = j
    keys = torch.tensor(list(last.keys()), device="cuda")
    rows = torch.tensor(list(last.values()), device="cuda")
    ref_v[keys] += out[rows]
    ref_c[keys] += 1
    ops.vote(votes, counts, stamp, dup, out, status=status)
    assert torch.equal(votes.view(torch.int32), ref_v.view(torch.int32))
    assert torch.equal(counts, ref_c)
    assert bool((stamp == -1).all()) and int(status.item()) == 0


@pytest.mark.parametrize("dt", list(DTYPES))
def test_vote_matches_index_put(dt):
    vote_scenario(dt)


def test_out_of_range_ids_are_skipped_and_flagged():
    votes = torch.zeros(10, 3, device="cuda")
    counts = torch.zeros(10, dtype=torch.int32, device="cuda")
    stamp = torch.full((10,), -1, dtype=torch.int32, device="cuda")
    status = ops.vote(votes, counts, stamp, torch.tensor([1, 10, -1, 2], device="cuda"), torch.ones(4, 3, device="cuda"))
    assert int(status.item()) == 4
    assert counts.tolist() == [0, 1, 1, 0, 0, 0, 0, 0, 0, 0]


# ---------------------------------------------------------------------------------------------------------------
# full resolution
# ---------------------------------------------------------------------------------------------------------------
def brute_nn(qpos, spos, chunk=4096):
    """Exact nearest search point, (dx dx + dy dy) + dz dz in fp32, ties to the lower index."""
    out = torch.empty(qpos.shape[0], dtype=torch.int64, device="cuda")
    ar = torch.arange(spos.shape[0], device="cuda")
    for s in range(0, qpos.shape[0], chunk):
        d = spos[None, :, :] - qpos[s:s + chunk, None, :]
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        m = d2.min(1, keepdim=True).values
        out[s:s + chunk] = torch.where(d2 == m, ar, spos.shape[0]).min(1).values
    return out


def full_res_oracle(votes, counts, pos, mode):
    """torch_geometric knn_interpolate(k=1) in its fp32 order, then argmax; torch on the GPU rounds every
    elementwise step on its own (no contraction across ops)."""
    has = counts > 0
    voted = torch.nonzero(has).squeeze(1)
    x = votes[voted]
    if mode == "interpolate_mean":
        x = x / counts[voted].unsqueeze(-1)
    q = torch.nonzero(~has).squeeze(1) if mode == "own_votes" else torch.arange(votes.shape[0], device="cuda")
    nn = brute_nn(pos[q], pos[voted])
    diff = pos[voted][nn] - pos[q]
    d2 = (diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1]) + diff[:, 2] * diff[:, 2]
    w = 1.0 / torch.clamp(d2, min=1e-16)
    y = (x[nn] * w[:, None]) / w[:, None]
    pred = torch.from_numpy(np.argmax(y.cpu().numpy(), 1)).cuda()
    if mode == "own_votes":
        full = torch.from_numpy(np.argmax(votes.cpu().numpy(), 1)).cuda()
        full[q] = pred
        return full
    return pred


def nn_case(N, K, voted_share, seed, far=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    pos = torch.rand(N, 3, generator=g, device="cuda") * torch.tensor([20.0, 20.0, 3.0], device="cuda")
    pos = (pos * 100).round() / 100                  # a 1 cm lattice: many exact distance ties
    counts = (torch.rand(N, generator=g, device="cuda") < voted_share).int() * \
        torch.randint(1, 4, (N,), generator=g, device="cuda", dtype=torch.int32)
    if far:                                          # an unvoted region far from every voted point
        counts[pos[:, 0] > 15] = 0
    votes = torch.randn(N, K, generator=g, device="cuda") * counts[:, None]
    votes[::97, 1] = votes[::97, 0]                  # exact ties between classes
    labels = torch.randint(0, K, (N,), generator=g, device="cuda")
    labels[::11] = -1
    return votes, counts, pos, labels


def nn_scenario(N=60_000, K=13):
    for mode, share, far in (("interpolate", 0.6, False), ("interpolate_mean", 0.3, True), ("own_votes", 0.5, True)):
        votes, counts, pos, labels = nn_case(N, K, share, seed=len(mode), far=far)
        cm = torch.zeros(K, K, dtype=torch.int64, device="cuda")
        pred, status = ops.full_res_predict(votes, counts, pos, labels=labels, cm=cm, ignore_label=-1, mode=mode)
        ref = full_res_oracle(votes, counts, pos, mode)
        assert torch.equal(pred, ref), (mode, int((pred != ref).sum()))
        keep = labels != -1
        assert torch.equal(cm, torch.bincount(K * labels[keep] + ref[keep], minlength=K * K).view(K, K)), mode
        assert int(status.item()) == 0


def test_full_resolution_modes_match_the_restated_interpolation():
    nn_scenario()


def test_full_resolution_five_million_points():
    N, K = 5_000_000, 13
    g = torch.Generator(device="cuda").manual_seed(9)
    pos = torch.rand(N, 3, generator=g, device="cuda") * torch.tensor([40.0, 40.0, 4.0], device="cuda")
    counts = torch.zeros(N, dtype=torch.int32, device="cuda")
    counts[torch.randperm(N, generator=g, device="cuda")[:20_000]] = 2
    votes = torch.randn(N, K, generator=g, device="cuda") * counts[:, None]
    pred, _ = ops.full_res_predict(votes, counts, pos)
    assert torch.equal(pred, full_res_oracle(votes, counts, pos, "interpolate"))


def test_zero_distance_rounding_is_torch_geometrics():
    """At d = 0, w = 1e16 and (x w) / w need not be x: a near-tie can flip, exactly as in knn_interpolate."""
    K = 2
    x = torch.tensor([[3.0000002, 3.0000000]], device="cuda")
    w = torch.tensor(1e16, device="cuda")
    y = (x * w) / w
    votes = torch.cat([x, torch.zeros(1, K, device="cuda")])
    counts = torch.tensor([1, 0], dtype=torch.int32, device="cuda")
    pos = torch.zeros(2, 3, device="cuda")
    pred, _ = ops.full_res_predict(votes, counts, pos)
    assert pred.tolist() == [int(np.argmax(y.cpu().numpy()[0]))] * 2


def test_empty_search_set_raises():
    with pytest.raises(ValueError, match="empty search set"):
        ops.full_res_predict(torch.zeros(4, 3, device="cuda"), torch.zeros(4, dtype=torch.int32, device="cuda"),
                             torch.zeros(4, 3, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------
# trackers
# ---------------------------------------------------------------------------------------------------------------
class _Dataset:
    def __init__(self, K, pos=None, y=None):
        self.num_classes = K
        self.INV_OBJECT_LABEL = {i: f"class{i}" for i in range(K)}
        self.test_data = types.SimpleNamespace(pos=pos, y=y)

    def has_labels(self, stage):
        return True


class _Model:
    is_multimodal = False

    def __init__(self, out, y, origin=None):
        self.out, self.y, self.inp = out, y, {"origin_id": origin}

    def get_output(self):
        return self.out

    def get_labels(self):
        return self.y

    def get_input(self):
        return self.inp


def np_metrics(cm):
    """The reference's formulas (metrics/confusion_matrix.py) on a numpy matrix."""
    cm = cm.astype(np.int64)
    tp = np.diagonal(cm)
    union = cm.sum(0) + cm.sum(1) - tp
    iou = 1e-8 + tp / (union + 1e-8)
    ex = union > 1e-3
    miou = np.sum(iou[ex]) / np.sum(ex) if np.sum(ex) else 0
    acc = float(np.trace(cm)) / max(int(cm.sum()), 1)
    re, pres = 0, 0
    for i in range(cm.shape[0]):
        t = np.sum(cm[i, :])
        if t:
            pres += 1
            re = re + cm[i][i] / max(1, t)
    return acc, (re / pres if pres else 0), miou, iou


def test_s3dis_tracker_reproduces_the_restated_reference():
    N, K, R = 30_000, 13, 8
    g = torch.Generator(device="cuda").manual_seed(5)
    pos = (torch.rand(N, 3, generator=g, device="cuda") * 10).cpu()
    y = torch.randint(0, K, (N,), generator=g, device="cuda").cpu()
    ds = _Dataset(K, pos, y)
    tr = S3DISTracker(ds, stage="test")
    votes = torch.zeros(N, K)
    counts = torch.zeros(N, dtype=torch.int32)
    batch_cm = np.zeros((K, K), dtype=np.int64)
    for r in range(R):
        ids = torch.randperm(N, generator=g, device="cuda")[:4000]      # overlapping samples, several runs
        out = torch.randn(4000, K, generator=g, device="cuda")
        lab = y.cuda()[ids].clone()
        lab[:400] = -1
        tr.track(_Model(out, lab, ids), full_res=True)
        keep = (lab != -1).cpu().numpy()
        batch_cm += np_confusion(lab.cpu().numpy()[keep], np_argmax(out)[keep], K)
        votes[ids.cpu()] += out.cpu()
        counts[ids.cpu()] += 1
    tr.finalise(full_res=True, vote_miou=True)
    m = tr.get_metrics(verbose=True)
    acc, macc, miou, iou = np_metrics(batch_cm)
    assert (tr.confusion_matrix == batch_cm).all()
    assert m["test_acc"] == 100 * acc and m["test_macc"] == 100 * macc and m["test_miou"] == 100 * miou
    assert m["test_miou_per_class"] == {i: "{:.2f}".format(100 * v) for i, v in enumerate(iou)}
    assert m["test_iou"] == {f"class{k}": v for k, v in enumerate(iou)}          # a fraction, as in the reference
    has = counts > 0
    vcm = np_confusion(y[has].numpy(), np.argmax(votes[has].numpy(), 1), K)
    _, _, vmiou, viou = np_metrics(vcm)
    assert m["test_vote_miou"] == vmiou * 100
    assert m["test_vote_iou"] == {f"class{k}": 100 * v for k, v in enumerate(viou)}
    full = full_res_oracle(votes.cuda(), counts.cuda(), pos.cuda(), "interpolate").cpu().numpy()
    fcm = np_confusion(y.numpy(), full, K)
    assert (tr.full_confusion_matrix.confusion_matrix == fcm).all()
    _, _, fmiou, fiou = np_metrics(fcm)
    assert m["test_full_vote_miou"] == fmiou * 100
    assert m["test_full_vote_iou"] == {f"class{k}": 100 * v for k, v in enumerate(fiou)}


def test_tracking_does_not_sync():
    N, K = 20_000, 13
    g = torch.Generator(device="cuda").manual_seed(6)
    pos = torch.rand(N, 3, generator=g, device="cuda")
    y = torch.randint(0, K, (N,), generator=g, device="cuda")
    batches = []
    for _ in range(3):
        ids = torch.randint(0, N, (3000,), generator=g, device="cuda")
        batches.append(_Model(torch.randn(3000, K, generator=g, device="cuda"), y[ids].clone(), ids))
    seg = SegmentationTracker(_Dataset(K), stage="val")
    s3 = S3DISTracker(_Dataset(K, pos, y), stage="test")
    s3.track(batches[0], full_res=True)                  # the first call moves the area to the device
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for b in batches:
            seg.track(b)
        for b in batches[1:]:
            s3.track(b, full_res=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert int(seg.confusion_matrix.sum()) == 9000


def test_s3dis_origin_ids_out_of_range_raise_at_finalise():
    N, K = 100, 4
    s3 = S3DISTracker(_Dataset(K, torch.rand(N, 3), torch.zeros(N, dtype=torch.int64)), stage="test")
    s3.track(_Model(torch.randn(3, K, device="cuda"), torch.zeros(3, dtype=torch.int64, device="cuda"),
                    torch.tensor([0, 5, N], device="cuda")), full_res=True)
    with pytest.raises(ValueError, match="origin id"):
        s3.finalise(full_res=True)
