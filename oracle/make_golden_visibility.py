"""Generate the Biasutti / depth-map visibility fixtures by EXECUTING THE REFERENCE (oracle; test
infrastructure).

Run in the build container only (needs the reference checkout, see oracle/ref_loader.py):
    PYTORCH_JIT=0 python -m oracle.make_golden_visibility
writes tests/golden/visibility_model_{biasutti_equirect_wrap,biasutti_scannet,depth_equirect}.npz
with the same saver and metadata as oracle/make_golden.py.
"""
import os
import sys

os.environ.setdefault("PYTORCH_JIT", "0")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import save  # noqa: E402


def _visibility_model_inputs():
    """the seeded inputs of oracle/make_golden.py::make_visibility_model_golden"""
    gen = torch.Generator().manual_seed(29)
    n = 7000
    xyz = (torch.rand(n, 3, generator=gen) - 0.5) * torch.tensor([12., 12., 4.])
    geo = torch.rand(n, 3, generator=gen)
    normals = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=1)
    img_xyz = torch.tensor([0.3, -0.2, 0.1])
    c2w = np.eye(4)
    a, b, c = -1.4, 0.1, 0.5
    rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    rz = np.array([[np.cos(c), -np.sin(c), 0], [np.sin(c), np.cos(c), 0], [0, 0, 1]])
    c2w[:3, :3] = rz @ ry @ rx
    c2w[:3, 3] = img_xyz.numpy()
    intr = np.eye(4, dtype=np.float32)
    intr[0, 0], intr[1, 1], intr[0, 2], intr[1, 2] = 250.0, 250.0, 159.5, 119.5
    return xyz, geo, normals, img_xyz, c2w, intr


def _points_at_distance(img_xyz, targets, rng):
    """points whose float32 camera distance (norm_cpu of xyz - img_xyz, visibility.py:130-145) is
    exactly each target: random directions, then a scan over radii in float32 steps"""
    from oracle import visibility_oracle as VO
    c = img_xyz.numpy().astype(np.float32)
    out = []
    for t in targets:
        for _ in range(200):
            u = rng.normal(size=3)
            u[2] = 0.2 * abs(u[2])
            u /= np.linalg.norm(u)
            r = np.float32(t) + np.arange(-4000, 4000, dtype=np.float64) * 2.0 ** -30
            p = (c[None, :] + (r[:, None] * u[None, :])).astype(np.float32)
            d, _, _, _ = VO.project_equirect(p, c, np.eye(3, dtype=np.float32), 64, 32, 0, 0, 0.0, 1e30)
            hit = np.nonzero(d == np.float32(t))[0]
            if hit.size:
                out.append(p[hit[0]])
                break
        else:
            raise RuntimeError(f"no point at distance {t!r}")
    return torch.from_numpy(np.stack(out))


def make_visibility_extra_golden(ref):
    """BiasuttiVisibility and DepthBasedVisibility .__call__ (visibility.py:1328-1500, 1779-1799)
    executed on the CPU (numba) path with the inputs of oracle/make_golden.py::make_visibility_model_golden.  The KeOps
    argKmin of k_nn_image_system (:1439-1444) is the dense stand-in of oracle/ref_loader.py (exact,
    ties by search-set index): `visibility.py` imported the name LazyTensor at load time, so the
    stand-in is bound on the module itself.  Besides the dict, the fixtures hold the projections,
    the executed k_nn_image_system neighbours' alpha (:1485-1489, torch CPU float32) and, for the
    depth case, the uint16 depth image (the test writes the PNG) and the executed
    read_s3dis_depth_map result."""
    import tempfile
    from PIL import Image
    vis = ref.visibility
    vis.LazyTensor = ref_loader.DenseLazyTensor
    xyz, geo, normals, img_xyz, c2w, intr = _visibility_model_inputs()
    opk = torch.tensor([0.05, -0.1, 0.7])

    def run(tag, model_cls, ctor, call, xyz, geo, normals, extra):
        model = model_cls(**ctor)
        out = model(xyz, img_xyz, linearity=geo[:, 0], planarity=geo[:, 1], scattering=geo[:, 2],
                    normals=normals, **call)
        proj_kw = {k: v for k, v in {**ctor, **call}.items()
                   if k not in ("k", "margin", "threshold", "depth_threshold", "depth_map_path")}
        idx, dist, xp, yp = vis.camera_projection_cpu(xyz, img_xyz, **proj_kw)
        stored = {k: v for k, v in ctor.items() if v is not None}        # None = the constructor default
        arrays = dict(xyz=xyz, img_xyz=img_xyz, geo=geo, normals=normals, ctor_keys=np.array(list(stored.keys())),
                      **{"ctor/" + k: np.asarray(v) for k, v in stored.items()},
                      **{"call/" + k: v for k, v in call.items() if k != "depth_map_path"},
                      **{"out/" + k: v for k, v in out.items()},
                      proj_idx=idx, dist=dist, x_proj=xp, y_proj=yp, **extra)
        if model_cls is vis.BiasuttiVisibility:
            nbr = vis.k_nn_image_system(xp, yp, k=ctor["k"], x_margin=ctor["margin"], x_width=ctor["img_size"][0])
            dnn = dist[nbr]
            dmin, dmax = dnn.min(dim=1).values, dnn.max(dim=1).values
            alpha = torch.exp(-((dist - dmin) / (dmax - dmin)) ** 2)
            arrays.update(alpha=alpha, threshold=alpha.mean() if ctor["threshold"] is None else
                          torch.tensor(ctor["threshold"], dtype=torch.float32), kth_nbr=nbr[:, -1])
        print(tag, {k: tuple(v.shape) for k, v in out.items()})
        save("visibility_model_" + tag, **arrays)

    run("biasutti_equirect_wrap", vis.BiasuttiVisibility,
        dict(k=75, margin=16, threshold=None, img_size=(512, 256), crop_top=0, crop_bottom=0, r_max=8, r_min=0.5,
             camera="s3dis_equirectangular"), dict(img_opk=opk), xyz, geo, normals, {})
    run("biasutti_scannet", vis.BiasuttiVisibility,
        dict(k=75, margin=None, threshold=0.6, img_size=(320, 240), r_max=8, r_min=0.3, camera="scannet"),
        dict(img_extrinsic=torch.from_numpy(np.linalg.inv(c2w)).float(), img_intrinsic_pinhole=torch.from_numpy(intr)),
        xyz, geo, normals, {})

    # depth map: per pixel the nearest projected depth, quantised to 1/512 m and shifted by up to
    # +-40/512 m, 10 % of the pixels empty (65535).  Three points sit at distances D - 1 ulp, D and
    # D + 1 ulp with D = 40/512 - fp32(0.05): against a depth of 40/512 their float32 differences round
    # to fp32(0.05) + 2**-28 (dropped), exactly fp32(0.05) (kept by a float32 comparison, dropped by a
    # float64 one) and fp32(0.05) - 2**-28 (kept)
    W, H = 512, 256
    ctor = dict(depth_threshold=0.05, img_size=(W, H), crop_top=0, crop_bottom=0, r_max=8, r_min=0.01,
                camera="s3dis_equirectangular")
    f32 = np.float32
    D = f32(40 / 512) - f32(0.05)
    assert f32(f32(40 / 512) - D) == f32(0.05)
    targets = [np.nextafter(D, f32(0)), D, np.nextafter(D, f32(1))]
    rng = np.random.default_rng(11)
    special = _points_at_distance(img_xyz, targets, rng)
    xyz_d = torch.cat([xyz, special])
    geo_d = torch.cat([geo, torch.rand(3, 3, generator=torch.Generator().manual_seed(3))])
    normals_d = torch.cat([normals, torch.nn.functional.normalize(torch.ones(3, 3), dim=1)])
    idx, dist, xp, yp = vis.camera_projection_cpu(
        xyz_d, img_xyz, img_opk=opk, **{k: v for k, v in ctor.items() if k != "depth_threshold"})
    assert set(range(xyz.shape[0], xyz.shape[0] + 3)) <= set(idx.tolist())
    dm = np.full((W, H), 2 ** 16 - 1, dtype=np.int64)
    px, py = xp.long().numpy(), yp.long().numpy()
    order = np.argsort(-dist.numpy(), kind="stable")                # nearest written last
    dm[px[order], py[order]] = np.rint(dist.numpy()[order].astype(np.float64) * 512).astype(np.int64)
    filled = dm != 2 ** 16 - 1
    dm[filled] += rng.integers(-40, 41, size=int(filled.sum()))
    dm[rng.random((W, H)) < 0.1] = 2 ** 16 - 1
    sp = np.nonzero(np.isin(idx.numpy(), np.arange(xyz.shape[0], xyz.shape[0] + 3)))[0]
    dm[px[sp], py[sp]] = 40
    dm = np.clip(dm, 0, 2 ** 16 - 1).astype(np.uint16)
    png = np.repeat(np.repeat(dm.T, 2, axis=0), 2, axis=1)          # [2H, 2W]: the reader resizes to (W, H)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "depth.png")
        Image.fromarray(png).save(path)
        depth_map = vis.read_s3dis_depth_map(path, img_size=(W, H), empty=-1)
        run("depth_equirect", vis.DepthBasedVisibility, ctor, dict(img_opk=opk, depth_map_path=path), xyz_d, geo_d,
            normals_d, dict(depth_png=png, depth_map=depth_map, special=np.arange(xyz.shape[0], xyz.shape[0] + 3)))


if __name__ == "__main__":
    make_visibility_extra_golden(ref_loader.load_reference())
