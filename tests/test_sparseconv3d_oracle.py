"""The float64 Lovász-softmax restatement (oracle/lovasz_oracle.py) against fixtures made by executing the
reference's metrics/lovasz_loss.py (tests/golden/lovasz_*.npz), and the loss bookkeeping of the reference's
sparse-conv models recorded in tests/golden/sparseconv3d_models.npz (CPU only)."""
import os

import numpy as np
import pytest

from oracle import lovasz_oracle as LO
from oracle.make_golden_sparseconv3d import MODEL_CASES

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
KINDS = ("tiefree", "ties", "ignored", "absent", "all", "list")


def load_lovasz(kind):
    z = np.load(os.path.join(GOLDEN, f"lovasz_{kind}.npz"))
    mode = str(z["classes_mode"])
    classes = [int(c) for c in z["classes"]] if mode == "list" else mode
    return z["probas"], z["labels"], classes, float(z["loss"]), z["grad"]


@pytest.mark.parametrize("kind", KINDS)
def test_lovasz_oracle_loss_matches_the_reference(kind):
    probas, labels, classes, loss, _ = load_lovasz(kind)
    got, _, _ = LO.lovasz_softmax(probas, labels, classes)
    # the reference computes in fp32 (errors, cumsum, Jaccard): a few ulp of fp32 per class term
    assert abs(got - loss) <= 1e-6 * max(1.0, abs(loss)), (got, loss)


@pytest.mark.parametrize("kind", [k for k in KINDS if k != "ties"])
def test_lovasz_oracle_gradient_matches_the_reference(kind):
    probas, labels, classes, _, grad = load_lovasz(kind)
    _, got, _ = LO.lovasz_softmax(probas, labels, classes)
    np.testing.assert_allclose(got, grad, rtol=1e-5, atol=1e-7)


def test_lovasz_oracle_tied_block_sums_match_the_reference():
    """On tied errors the gradient of one element depends on the order of the tie; the sum over a tied block of
    grad * d|fg - p| / dp does not."""
    probas, labels, classes, _, grad = load_lovasz("ties")
    _, got, _ = LO.lovasz_softmax(probas, labels, classes)
    for c in range(probas.shape[1]):
        for blk in LO.sorted_blocks(probas, labels, c):
            s = -np.sign((labels[blk] == c) - probas[blk, c].astype(np.float64))
            assert abs(float((got[blk, c] * s).sum() - (grad[blk, c] * s).sum())) <= 1e-6, (c, blk)


def test_lovasz_oracle_edges():
    p = np.full((4, 3), 1 / 3)
    assert LO.lovasz_softmax(p, np.full(4, -1))[0] == 0.0                        # no valid point
    assert LO.lovasz_softmax(p[:1], np.array([2]))[0] == pytest.approx(2 / 3)    # a single valid point
    assert LO.lovasz_softmax(p, np.array([0, 1, 0, 1]), classes=[2])[0] == pytest.approx(1 / 3)
    loss, grad, _ = LO.lovasz_softmax(p, np.array([-1, -1, 0, 0]), classes=[])   # no kept class
    assert loss == 0.0 and not grad.any()


def test_model_fixture_losses_add_up():
    """loss_seg is the sum of the recorded terms, with LateFeatureFusion's auxiliary cross-entropy counted twice
    (models/segmentation/multimodal/sparseconv3d.py:141-181)."""
    z = np.load(os.path.join(GOLDEN, "sparseconv3d_models.npz"))
    for case, cls_name, opts in MODEL_CASES:
        if cls_name == "LateLogitFusion" or (not opts.get("use_cross_entropy", True) and
                                             (opts.get("loss_no3d") or opts.get("loss_3d"))):
            continue                                  # an unrecorded term: nothing to add up
        names = [str(n) for n in z[f"{case}/loss_names"]]
        total = sum(float(z[f"{case}/{n}"]) * (2 if n.startswith("loss_cross_entropy_") else 1)
                    for n in names if n != "loss_seg")
        assert abs(total - float(z[f"{case}/loss_seg"])) <= 1e-5 * abs(total), (case, names)
