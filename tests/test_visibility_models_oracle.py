"""CPU side of the Biasutti and depth-map visibility models: the numpy restatements of
oracle/visibility_models_oracle.py against fixtures of the executed reference
(tests/golden/visibility_model_{biasutti_*,depth_*}.npz), the image-plane k-NN against the dense
KeOps stand-in and cKDTree, the depth PNG reader, and the k range of dva_knn_grid."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from deepviewagg_b200 import _lib
from oracle import visibility_models_oracle as VO
from oracle.ref_loader import DenseLazyTensor

BAND_ULP = 4


def fixture(tag):
    z = np.load(os.path.join(GOLDEN, f"visibility_model_{tag}.npz"))
    ctor = {k: (z["ctor/" + k].tolist() if z["ctor/" + k].ndim else z["ctor/" + k].item())
            for k in z["ctor_keys"].tolist()}
    ctor["img_size"] = tuple(ctor["img_size"])
    return z, ctor


def ulp_dist(a, b):
    a = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    b = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(a - b)


def in_band(alpha, thr, ulps=BAND_ULP):
    """alpha within `ulps` float32 steps of the threshold (both sides)"""
    return np.isfinite(alpha) & (ulp_dist(alpha, np.full_like(alpha, thr)) <= ulps)


@pytest.mark.parametrize("tag", ["biasutti_equirect_wrap", "biasutti_scannet"])
def test_biasutti_oracle_vs_reference(tag):
    z, ctor = fixture(tag)
    margin, thr_arg = ctor.get("margin"), ctor.get("threshold")
    nbr, _ = VO.image_knn(z["x_proj"], z["y_proj"], ctor["k"], margin, ctor["img_size"][0])
    assert np.array_equal(nbr[:, -1], z["kth_nbr"])                       # integers exact
    idx2, alpha, thr = VO.biasutti_visibility(z["x_proj"], z["y_proj"], z["dist"], ctor["img_size"], ctor["k"],
                                              margin, thr_arg, neighbors=nbr)
    ref_alpha = z["alpha"]
    assert np.array_equal(np.isnan(alpha), np.isnan(ref_alpha))
    fin = np.isfinite(ref_alpha)
    assert ulp_dist(alpha[fin], ref_alpha[fin]).max() <= 2
    # float64 mean rounded to float32 vs the reference's float32 mean: a few ulps apart at most
    assert ulp_dist(thr, z["threshold"]) <= BAND_ULP
    kept = np.zeros(alpha.shape[0], bool)
    kept[idx2] = True
    ref_kept = np.isin(z["proj_idx"], z["out/idx"])
    band = in_band(ref_alpha, z["threshold"])
    assert np.array_equal(kept[~band], ref_kept[~band])
    # the assembled dict on the points both sides keep
    out = VO.model_visibility("BiasuttiVisibility", z["xyz"], z["img_xyz"], z["geo"][:, 0], z["geo"][:, 1],
                              z["geo"][:, 2], z["normals"], **ctor,
                              **{k[5:]: z[k] for k in z.files if k.startswith("call/")})
    both = np.intersect1d(out["idx"], z["out/idx"])
    a = np.searchsorted(out["idx"], both)
    b = np.searchsorted(z["out/idx"], both)
    for k in ("x", "y", "depth"):
        assert np.array_equal(out[k][a], z["out/" + k][b]), k
    assert np.abs(out["features"][a] - z["out/features"][b]).max() <= 1e-6
    assert len(np.setxor1d(out["idx"], z["out/idx"])) == int((band & (kept != ref_kept)).sum())


def test_depth_oracle_vs_reference():
    z, ctor = fixture("depth_equirect")
    call = {k[5:]: z[k] for k in z.files if k.startswith("call/")}
    out = VO.model_visibility("DepthBasedVisibility", z["xyz"], z["img_xyz"], z["geo"][:, 0], z["geo"][:, 1],
                              z["geo"][:, 2], z["normals"], depth_map=z["depth_map"], **ctor, **call)
    for k in ("idx", "x", "y", "depth"):
        assert out[k].dtype == z["out/" + k].dtype and np.array_equal(out[k], z["out/" + k]), k
    assert np.abs(out["features"] - z["out/features"]).max() <= 1e-6
    # the three threshold-boundary points: |d_real - dist| = fp32(0.05) + 2**-28, fp32(0.05), fp32(0.05) - 2**-28;
    # the reference keeps the middle one, i.e. it compares in float32
    kept = np.isin(z["special"], z["out/idx"])
    assert kept.tolist() == [False, True, True]
    assert (z["depth_map"] == -1).any() and (z["depth_png"] == 65535).any()


def test_read_s3dis_depth_map_matches_reference():
    PIL = pytest.importorskip("PIL.Image")
    from deepviewagg_b200.core.multimodal.visibility import read_s3dis_depth_map
    z, ctor = fixture("depth_equirect")
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "depth.png")
        PIL.fromarray(z["depth_png"]).save(path)
        dm = read_s3dis_depth_map(path, img_size=ctor["img_size"])
        assert dm.dtype == torch.float32 and tuple(dm.shape) == ctor["img_size"]
        assert np.array_equal(dm.numpy(), z["depth_map"])
        full = read_s3dis_depth_map(path, empty=-3)
        assert tuple(full.shape) == (z["depth_png"].shape[1], z["depth_png"].shape[0])
        assert np.array_equal(full.numpy() == -3, z["depth_png"].T == 65535)


def _dense_reference_knn(xp, yp, k, x_margin, x_width):
    """k_nn_image_system (visibility.py:1413-1458) with the dense LazyTensor stand-in"""
    q = torch.stack((torch.from_numpy(xp).float(), torch.from_numpy(yp).float())).t()
    xp_t = torch.from_numpy(xp)
    left = torch.where(xp_t <= x_margin)[0]
    right = torch.where(xp_t >= (x_width - x_margin))[0]
    off = torch.Tensor([[x_width, 0]]).float()
    s = torch.cat((q, q[left] + off, q[right] - off))
    d = ((DenseLazyTensor(q[:, None, :]) - DenseLazyTensor(s[None, :, :])) ** 2).sum(dim=2)
    nbr = d.argKmin(k, dim=1)
    n, nl = q.shape[0], left.shape[0]
    is_l = (nbr >= n) & (nbr < n + nl)
    nbr[is_l] = left[nbr[is_l] - n]
    is_r = nbr >= n + nl
    nbr[is_r] = right[nbr[is_r] - n - nl]
    return nbr.numpy()


def test_image_knn_wrap_vs_dense_and_ckdtree():
    from scipy.spatial import cKDTree
    z, ctor = fixture("biasutti_equirect_wrap")
    xp, yp = z["x_proj"][:2500], z["y_proj"][:2500]
    W, margin, k = ctor["img_size"][0], ctor["margin"], ctor["k"]
    nbr, d2 = VO.image_knn(xp, yp, k, margin, W)
    assert np.array_equal(nbr, _dense_reference_knn(xp, yp, k, margin, W))
    # k-th distance against scipy on the same float32 search set
    xy = np.stack([xp.astype(np.float32), yp.astype(np.float32)], 1)
    off = np.array([np.float32(W), 0], np.float32)
    s = np.concatenate([xy, xy[xp <= margin] + off, xy[xp >= W - margin] - off]).astype(np.float64)
    dk, _ = cKDTree(s).query(xy.astype(np.float64), k=k)
    assert np.allclose(d2[:, -1], dk[:, -1] ** 2, rtol=1e-6, atol=0)
    # the candidate path (large search sets) gives the same rows as the brute force
    nbr_c, d2_c = VO.image_knn(xp, yp, k, margin, W, exact_below=0)
    assert np.array_equal(nbr_c, nbr) and np.array_equal(d2_c, d2)


def test_image_knn_clamps_k_to_search_set():
    xp = np.array([1.0, 2.0, 5.0, 509.0])
    yp = np.array([3.0, 3.0, 3.0, 3.0])
    nbr, _ = VO.image_knn(xp, yp, 75, 4, 512)
    assert nbr.shape == (4, 7)                                 # 4 points + 2 left copies + 1 right copy
    assert np.array_equal(nbr, _dense_reference_knn(xp, yp, 7, 4, 512))


def test_knn_grid_k_range_refused_without_launch():
    lib = _lib.load()
    n0 = _lib.launch_count()
    for k in (0, 129, -1):
        rc = lib.dva_knn_grid(None, None, None, None, 10, k, 0.0, 0.0, 0.0, 1.0, 1, 1, 1, None, None, None)
        assert rc == _lib.DVA_EUNSUPPORTED, k
        assert b"k must be in [1, 128]" in lib.dva_last_error()
    # k in range passes the k check and stops at the null pointers
    for k in (1, 64, 65, 128):
        assert lib.dva_knn_grid(None, None, None, None, 10, k, 0.0, 0.0, 0.0, 1.0, 1, 1, 1, None, None,
                                None) == _lib.DVA_EINVAL, k
    assert _lib.launch_count() == n0


def test_knn_grid_python_checks_k():
    from deepviewagg_b200.core.multimodal.mapping import knn_grid
    pos = torch.zeros(200, 3)
    if torch.cuda.is_available():
        pos = pos.cuda()
    else:
        pytest.skip("knn_grid argument checks run after the CUDA-tensor check")
    for k in (0, 129):
        with pytest.raises(ValueError, match=r"\[1, 128\]"):
            knn_grid(pos, k)
    with pytest.raises(ValueError, match="at least k=128"):
        knn_grid(pos[:100], 128)


def test_map_images_methods():
    from deepviewagg_b200.core.multimodal.mapping import MapImages
    for m in ("SplattingVisibility", "DepthBasedVisibility", "BiasuttiVisibility"):
        assert MapImages(method=m).method == m
    with pytest.raises(NotImplementedError):
        MapImages(method="NoSuchVisibility")
