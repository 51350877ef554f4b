"""The numpy restatement of the No3D models (oracle/no3d_oracle.py) against the fixtures the
reference produced (oracle/make_golden_no3d.py), and the query / search brute-force k-NN oracle.
No GPU needed."""
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import no3d_oracle as O

SAMPLES = ("main", "ties", "noseen", "allseen")
CLASSES = ("No3DFeatureFusion", "No3DLogitFusion", "No3DImageFeatureFusion", "No3DImageLogitFusion")


def load_no3d(kind):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"no3d_{kind}.npz"), allow_pickle=False)
    return {k: z[k] for k in z.files}


def fixture_inputs(g, cls_name):
    settings, maps = [], []
    s = 0
    while f"s{s}_pid" in g:
        settings.append({k: g[f"s{s}_{k}"] for k in ("pid", "iid", "pix", "feat", "size")})
        maps.append(g[f"{cls_name}/map{s}"])
        s += 1
    sd = {k[len(f"sd/{cls_name}/"):]: v for k, v in g.items() if k.startswith(f"sd/{cls_name}/")}
    return settings, maps, sd, g.get(f"{cls_name}/x3d")


def classes_of(g):
    return [c for c in CLASSES if f"{c}/train/output" in g]


@pytest.mark.parametrize("kind", SAMPLES)
def test_oracle_matches_reference_fixtures(kind):
    g = load_no3d(kind)
    classes = classes_of(g)
    assert len(classes) == (2 if kind == "noseen" else 4)
    for cls_name in classes:
        settings, maps, sd, x3d = fixture_inputs(g, cls_name)
        for mode in ("train", "eval"):
            out, loss, labels = O.no3d_forward(cls_name, mode == "train", g["pos"], g["labels"], settings, maps,
                                               sd, x3d)
            ref = g[f"{cls_name}/{mode}/output"]
            what = f"{kind} {cls_name} {mode}"
            assert np.abs(out - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), what
            assert np.array_equal(labels, g[f"{cls_name}/{mode}/labels"]), what
            ref_loss = float(g[f"{cls_name}/{mode}/loss"])
            if np.isnan(ref_loss):
                assert np.isnan(loss), what
            else:
                assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), what


def test_fixtures_cover_the_cases():
    """ties: unseen points equidistant from two seen points, and duplicated seen points;
    noseen: no point seen; allseen: no unseen point; main: a whole unseen region."""
    seen = {k: load_no3d(k)["seen"] for k in SAMPLES}
    assert not seen["noseen"].any() and seen["allseen"].all()
    assert 0.2 < seen["main"].mean() < 0.8
    g = load_no3d("ties")
    pos, s = g["pos"], g["seen"]
    _, d2 = O.knn_query_bruteforce(pos[~s], pos[s], 2)
    assert (d2[:, 0] == d2[:, 1]).sum() >= 10
    sp = pos[s]
    assert len({tuple(p) for p in sp.tolist()}) < sp.shape[0]


def test_knn_query_bruteforce_ties_and_self():
    rng = np.random.default_rng(3)
    search = rng.integers(0, 4, (200, 3)).astype(np.float32)        # many exact ties
    query = rng.integers(0, 4, (50, 3)).astype(np.float32) + 0.5
    nbr, d2 = O.knn_query_bruteforce(query, search, 7)
    full = ((query[:, None, :] - search[None]) ** 2).sum(-1)
    for i in range(query.shape[0]):
        order = sorted(range(search.shape[0]), key=lambda j: (full[i, j], j))[:7]
        assert nbr[i].tolist() == order
        assert np.array_equal(d2[i], full[i, order].astype(np.float32))
    from oracle.neighborhood_oracle import knn_bruteforce
    a, _ = knn_bruteforce(search, 5)
    b, _ = O.knn_query_bruteforce(search, search, 5)
    assert np.array_equal(a, b)
