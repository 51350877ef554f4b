"""Biasutti and depth-map visibility on the GPU: the grid k-NN for 64 < k <= 128 and for planar
(image-plane) inputs, k_nn_image_system, the two VisibilityModel subclasses against the executed
reference (tests/golden/visibility_model_{biasutti_*,depth_*}.npz) and the oracle, and MapImages
with both methods."""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import visibility_models_oracle as VO
from test_visibility_models_oracle import BAND_ULP, fixture, in_band

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cell_size", [None, 0.05, 0.4, 3.0])
def test_knn_grid_wide_k_matches_bruteforce(cell_size):
    """k = 65, 75, 128: indices and d2 exact.  At cell_size 0.05 the 128th neighbour lies beyond the
    6 shells the kernel visits, so every query takes the exhaustive scan."""
    from deepviewagg_b200.core.multimodal.mapping import knn_grid
    from oracle.neighborhood_oracle import knn_bruteforce
    g = load_golden("neighborhood_features")
    pos = g["pos"].cuda()
    for k in (65, 75, 128):
        nbr, d2 = knn_grid(pos, k, cell_size=cell_size, return_dist2=True)
        want, d2_ref = knn_bruteforce(g["pos"].numpy(), k)
        assert np.array_equal(nbr.cpu().numpy(), want), k
        assert np.array_equal(d2.cpu().numpy(), d2_ref), k
    if cell_size == 0.05:
        reach = 6 * 0.05
        assert (d2_ref[:, -1] > reach * reach).all()


def test_knn_grid_planar_million_points_sampled():
    """1 M planar points (z = 0): uniform field, a dense clump, exact duplicates and far outliers
    (the outliers' neighbours lie far beyond 6 shells: exhaustive scan); k = 75."""
    from deepviewagg_b200.core.multimodal.mapping import knn_grid
    gen = torch.Generator().manual_seed(8)
    n, k = 1_000_000, 75
    xy = torch.rand(n, 2, generator=gen) * torch.tensor([2048.0, 1024.0])
    xy[:20000] = torch.tensor([700.0, 300.0]) + 0.5 * torch.randn(20000, 2, generator=gen)   # clump
    xy[20000:20300] = xy[20300:20600]                                                       # duplicates
    xy[20600:20700] = xy[20300]                                                             # 101 copies of one point
    xy[20700:20720] = 1e5 + 1e4 * torch.rand(20, 2, generator=gen)                          # outliers
    pos = torch.cat([xy, torch.zeros(n, 1)], 1)
    nbr, d2 = knn_grid(pos.cuda(), k, return_dist2=True)
    nbr, d2 = nbr.cpu().numpy(), d2.cpu().numpy()
    assert (np.diff(d2, axis=1) >= 0).all()
    p = xy.numpy().astype(np.float32)
    q = np.concatenate([np.arange(0, 20720, 37), np.arange(20700, 20720),
                        torch.randint(0, n, (400,), generator=gen).numpy()])
    for i in q.tolist():
        d = p[i] - p
        dd = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + np.float32(0) * np.float32(0)
        cand = np.argpartition(dd, k)[:k + 1]
        cand = np.unique(np.concatenate([cand, np.nonzero(dd <= dd[cand].max())[0]]))
        want = cand[np.lexsort((cand, dd[cand]))][:k]
        assert np.array_equal(nbr[i], want), i
        assert np.array_equal(d2[i], dd[want]), i


@pytest.mark.parametrize("tag", ["biasutti_equirect_wrap", "biasutti_scannet"])
def test_k_nn_image_system_equals_oracle(tag):
    from deepviewagg_b200.core.multimodal.visibility import k_nn_image_system
    z, ctor = fixture(tag)
    margin = ctor.get("margin")
    nbr = k_nn_image_system(torch.from_numpy(z["x_proj"]).cuda(), torch.from_numpy(z["y_proj"]).cuda(), k=ctor["k"],
                            x_margin=margin, x_width=ctor["img_size"][0])
    want, _ = VO.image_knn(z["x_proj"], z["y_proj"], ctor["k"], margin, ctor["img_size"][0])
    assert np.array_equal(nbr.cpu().numpy(), want)
    assert np.array_equal(nbr[:, -1].cpu().numpy(), z["kth_nbr"])


def _run_model(cls, z, ctor, **extra):
    call = {k[5:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("call/")}
    geo = torch.from_numpy(z["geo"]).cuda()
    model = cls(**ctor)
    return model(torch.from_numpy(z["xyz"]).cuda(), torch.from_numpy(z["img_xyz"]), linearity=geo[:, 0],
                 planarity=geo[:, 1], scattering=geo[:, 2], normals=torch.from_numpy(z["normals"]).cuda(), **call,
                 **extra)


def _check_dict_exact(out, z):
    for k in ("idx", "x", "y", "depth"):
        ref = torch.from_numpy(z["out/" + k])
        assert out[k].dtype == ref.dtype and torch.equal(out[k].cpu(), ref), k
    f, ref = out["features"].cpu(), torch.from_numpy(z["out/features"])
    assert f.dtype == torch.float32 and f.shape == ref.shape
    assert (f - ref).abs().max() <= 1e-6
    assert torch.equal(f[:, :4], ref[:, :4])


def test_depth_visibility_dict_vs_reference():
    from deepviewagg_b200.core.multimodal import visibility as V
    z, ctor = fixture("depth_equirect")
    out = _run_model(V.DepthBasedVisibility, z, ctor, depth_map=torch.from_numpy(z["depth_map"]).cuda())
    _check_dict_exact(out, z)
    PIL = pytest.importorskip("PIL.Image")
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "depth.png")
        PIL.fromarray(z["depth_png"]).save(path)
        _check_dict_exact(_run_model(V.DepthBasedVisibility, z, ctor, depth_map_path=path), z)


def _check_band(out, ref_idx, alpha_by_idx, thr):
    """kept sets identical except for points whose alpha is within BAND_ULP of the threshold"""
    got = set(out["idx"].cpu().tolist())
    diff = got.symmetric_difference(set(ref_idx.tolist()))
    band_ids = {int(i) for i, a in alpha_by_idx.items() if in_band(np.float32([a]), thr)[0]}
    assert diff <= band_ids, sorted(diff - band_ids)[:10]
    return diff


@pytest.mark.parametrize("tag", ["biasutti_equirect_wrap", "biasutti_scannet"])
def test_biasutti_visibility_dict_vs_reference(tag):
    from deepviewagg_b200.core.multimodal import visibility as V
    z, ctor = fixture(tag)
    out = _run_model(V.BiasuttiVisibility, z, ctor)
    assert out["x"].dtype == torch.float64 and out["y"].dtype == torch.float64
    alpha = dict(zip(z["proj_idx"].tolist(), z["alpha"].tolist()))
    diff = _check_band(out, z["out/idx"], alpha, z["threshold"])
    both = np.intersect1d(out["idx"].cpu().numpy(), z["out/idx"])
    a = np.searchsorted(out["idx"].cpu().numpy(), both)
    b = np.searchsorted(z["out/idx"], both)
    for k in ("x", "y", "depth"):
        assert np.array_equal(out[k].cpu().numpy()[a], z["out/" + k][b]), k
    assert np.abs(out["features"].cpu().numpy()[a] - z["out/features"][b]).max() <= 1e-6
    print(f"{tag}: {len(diff)} points in the +-{BAND_ULP} ulp band decided differently")


def test_biasutti_visibility_300k_vs_oracle():
    """300 k points in a room around an equirectangular camera, margin 32, k = 75, against the
    oracle (float64-mean threshold on both sides)."""
    from deepviewagg_b200.core.multimodal import visibility as V
    sys_path_tools = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools")
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_visibility", os.path.join(sys_path_tools, "bench_visibility.py"))
    bv = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bv)
    xyz = bv.room_scene(300_000, seed=4)
    cam, opk = torch.tensor([6.0, 4.5, 1.5]), torch.tensor([0.0, 0.0, 0.3])
    W, H = 2048, 1024
    _, dist, xp, yp = V.camera_projection(xyz.cuda(), cam, img_opk=opk, img_size=(W, H), r_max=30, r_min=0.5)
    xp_n, yp_n, d_n = xp.cpu().numpy(), yp.cpu().numpy(), dist.cpu().numpy()
    nbr = V.k_nn_image_system(xp, yp, k=75, x_margin=32, x_width=W)
    want, _ = VO.image_knn(xp_n, yp_n, 75, 32, W)
    assert np.array_equal(nbr.cpu().numpy(), want)
    idx2, _, _ = V.visibility_biasutti(xp, yp, dist, img_size=(W, H), k=75, margin=32)
    ref_idx, alpha, thr = VO.biasutti_visibility(xp_n, yp_n, d_n, (W, H), 75, 32, None, neighbors=want)
    _check_band({"idx": idx2}, ref_idx, dict(enumerate(alpha.tolist())), thr)
    assert 0.2 * len(xp_n) < len(ref_idx) < 0.95 * len(xp_n)


def test_biasutti_nan_small_and_empty():
    from deepviewagg_b200.core.multimodal.visibility import BiasuttiVisibility, visibility_biasutti
    dev = "cuda"
    gen = torch.Generator().manual_seed(1)
    xp = (torch.rand(500, generator=gen) * 200).double().to(dev)
    yp = (torch.rand(500, generator=gen) * 100).double().to(dev)
    d = (torch.rand(500, generator=gen) * 5 + 1).to(dev)
    # a group of 80 far-away projections sharing one depth: their alpha is 0/0 = NaN
    xp[:80] = 150.0 + torch.arange(80, device=dev).double() * 1e-3
    yp[:80] = 1000.0
    d[:80] = 2.5
    idx, _, _ = visibility_biasutti(xp, yp, d, img_size=(200, 100), k=75, threshold=0.0)
    assert not (idx < 80).any() and (idx >= 80).sum() == 420          # NaN never kept, alpha >= 0 otherwise
    idx, _, _ = visibility_biasutti(xp, yp, d, img_size=(200, 100), k=75)
    assert idx.numel() == 0                                            # NaN mean: nothing kept
    # n < k: every point is a neighbour of every point
    idx, x, y = visibility_biasutti(xp[100:110], yp[100:110], d[100:110], img_size=(200, 100), k=75)
    ref, _, _ = VO.biasutti_visibility(xp[100:110].cpu().numpy(), yp[100:110].cpu().numpy(),
                                       d[100:110].cpu().numpy(), (200, 100), 75)
    assert np.array_equal(idx.cpu().numpy(), ref) and torch.equal(x, xp[100:110][idx])
    # an image that keeps nothing
    z, ctor = fixture("biasutti_scannet")
    ctor["threshold"] = 2.0
    out = _run_model(BiasuttiVisibility, z, ctor)
    assert out["idx"].numel() == 0 and out["features"].shape[0] == 0


def _scene():
    g = load_golden("zbuffer_nocrop")
    W, H = [int(v) for v in g["size"]]
    cams = torch.stack([g["img_xyz"], g["img_xyz"] + torch.tensor([1.5, -0.7, 0.1]), torch.tensor([50., 50., 50.])])
    opk = torch.stack([g["img_opk"], g["img_opk"] * 0.5, g["img_opk"]])
    return g["xyz"], cams, opk, W, H


def _depth_maps(xyz, cams, opk, W, H):
    """per image: the nearest projected depth per pixel + 2 cm (-1 where nothing projects)"""
    from deepviewagg_b200.core.multimodal.visibility import camera_projection
    maps = torch.full((cams.shape[0], W, H), -1.0, device="cuda")
    for i in range(cams.shape[0]):
        _, d, xp, yp = camera_projection(xyz.cuda(), cams[i], img_opk=opk[i], img_size=(W, H), r_max=8, r_min=0.5)
        flat = torch.full((W * H,), float("inf"), device="cuda")
        flat.scatter_reduce_(0, xp.long() * H + yp.long(), d, reduce="amin")
        m = torch.isfinite(flat)
        maps[i].view(-1)[m] = flat[m] + 0.02
    return maps


@pytest.mark.parametrize("method", ["DepthBasedVisibility", "BiasuttiVisibility"])
def test_map_images_new_methods_equal_per_image_loop(method):
    from deepviewagg_b200.core.multimodal import visibility as V
    from deepviewagg_b200.core.multimodal.image import ImageMapping, SameSettingImageData
    from deepviewagg_b200.core.multimodal.mapping import MapImages
    from deepviewagg_b200.utils.multimodal import lexargunique
    from test_gpu_integer import _mapping_equal
    xyz, cams, opk, W, H = _scene()
    params = dict(depth_threshold=0.05) if method == "DepthBasedVisibility" else dict(k=75, margin=16)
    extras = {}
    if method == "DepthBasedVisibility":
        extras["depth_map"] = _depth_maps(xyz, cams, opk, W, H)
    images = SameSettingImageData(pos=cams, opk=opk, ref_size=(W // 2, H // 2), proj_upscale=2, downscale=1, **extras)
    mi = MapImages(method=method, r_max=8, r_min=0.5, **params)
    out = mi(xyz, images)
    out2 = mi(xyz, images)
    assert out.num_views == 2
    _mapping_equal(out.mappings, out2.mappings)
    assert torch.equal(out.mappings.features.cpu(), out2.mappings.features.cpu())
    model = getattr(V, method)(img_size=(W, H), r_max=8, r_min=0.5, **params)
    pid, iid, pix, feat = [], [], [], []
    for i in range(2):
        kw = {"depth_map": extras["depth_map"][i]} if extras else {}
        o = model(xyz.cuda(), cams[i], img_opk=opk[i], **kw)
        px, py = o["x"].long() // 2, o["y"].long() // 2
        p = o["idx"]
        u = lexargunique(p, px, py)
        pid.append(p[u]); iid.append(torch.full((u.numel(),), i, device="cuda"))
        pix.append(torch.stack([px[u], py[u]], 1).short()); feat.append(o["features"][u])
    ref = ImageMapping.from_dense(torch.cat(pid), torch.cat(iid), torch.cat(pix), torch.cat(feat),
                                  num_points=xyz.shape[0])
    _mapping_equal(out.mappings, ref)


def test_map_images_depth_needs_depth_maps():
    from deepviewagg_b200.core.multimodal.image import SameSettingImageData
    from deepviewagg_b200.core.multimodal.mapping import MapImages
    xyz, cams, opk, W, H = _scene()
    images = SameSettingImageData(pos=cams, opk=opk, ref_size=(W // 2, H // 2), proj_upscale=2, downscale=1)
    with pytest.raises(ValueError, match="read_s3dis_depth_map"):
        MapImages(method="DepthBasedVisibility", r_max=8, r_min=0.5)(xyz, images)
