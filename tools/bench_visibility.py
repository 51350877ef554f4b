"""Times the image-plane k-NN and the Biasutti visibility model on a synthetic equirectangular scene.

    python tools/bench_visibility.py [--out profiles/h100_visibility.jsonl] [--baseline-lib PATH]

One JSON line per measurement (plus one with the GPU name and power limit, read in the same run):
  * knn_grid alone on the wrapped search set of a 2048 x 1024 image (margin 32, k = 75) and the
    whole BiasuttiVisibility.__call__ (projection, k-NN, alpha, threshold, features), at 100 k and
    1 M projected points;
  * at 100 k, a dense GPU brute force of the same k-NN (chunked torch.cdist + topk, the algorithm
    class of the KeOps argKmin the reference runs);
  * knn_grid at k = 20 on the 300 k-point cloud of tests/test_gpu_neighborhood.py; with
    --baseline-lib (a libdva_b200.so built from another revision) the same call through that
    library, alternated with this one, so that the k <= 64 path can be compared across revisions.
Times are CUDA events around `--iters` calls after `--warmup` calls (median and min reported).
"""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return {"median_ms": round(ts[len(ts) // 2], 3), "min_ms": round(ts[0], 3), "iters": iters}


def room_scene(n, seed):
    """points on the walls, floor and ceiling of a 12 x 9 x 3 m room plus clutter, camera inside"""
    gen = torch.Generator().manual_seed(seed)
    u = torch.rand(n, 3, generator=gen)
    face = torch.randint(0, 7, (n,), generator=gen)
    size = torch.tensor([12.0, 9.0, 3.0])
    p = u * size
    for f, (ax, val) in enumerate([(0, 0.0), (0, 12.0), (1, 0.0), (1, 9.0), (2, 0.0), (2, 3.0)]):
        p[face == f, ax] = val
    p += 0.005 * torch.randn(n, 3, generator=gen)
    return p


def cloud_300k():
    """the 300 k-point cloud of tests/test_gpu_neighborhood.py::test_knn_grid_large_cloud_sampled_against_bruteforce"""
    gen = torch.Generator().manual_seed(3)
    n = 300_000
    uv = torch.rand(n, 2, generator=gen) * torch.tensor([40.0, 25.0])
    z = torch.where(torch.rand(n, generator=gen) < 0.6, 0.03 * torch.randn(n, generator=gen),
                    3.0 + 0.5 * torch.sin(uv[:, 0]) + 0.03 * torch.randn(n, generator=gen))
    pos = torch.cat([uv, z[:, None]], 1)
    pos[:5000] = torch.tensor([5.0, 5.0, 1.0]) + 0.01 * torch.randn(5000, 3, generator=gen)
    pos[5000:5010] = 500.0 + 100 * torch.rand(10, 3, generator=gen)
    return pos


def search_set(xp, yp, W, margin):
    xy = torch.stack((xp.float(), yp.float()), 1)
    off = torch.tensor([[float(W), 0.0]], device=xy.device)
    left = torch.nonzero(xp <= margin).view(-1)
    right = torch.nonzero(xp >= W - margin).view(-1)
    return torch.cat((xy, xy[left] + off, xy[right] - off))


def dense_knn(q, s, k, chunk=4096):
    out = torch.empty((q.shape[0], k), dtype=torch.int64, device=q.device)
    for i in range(0, q.shape[0], chunk):
        d = torch.cdist(q[i:i + chunk], s)
        out[i:i + chunk] = torch.topk(d, k, dim=1, largest=False).indices
    return out


def load_lib(path):
    from deepviewagg_b200 import _lib
    lib = ctypes.CDLL(os.path.abspath(path))
    for name, (res, args) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_visibility.jsonl"))
    ap.add_argument("--baseline-lib", default="")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_visibility measures on a CUDA device; there is no CPU fallback"
    from bench import gpu_identity
    from deepviewagg_b200 import _lib
    from deepviewagg_b200.core.multimodal import visibility as V
    from deepviewagg_b200.core.multimodal.mapping import knn_grid

    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    ident = gpu_identity(0)
    emit({"gpu": ident})
    W, H, margin, k = 2048, 1024, 32, 75
    cam = torch.tensor([6.0, 4.5, 1.5])
    opk = torch.tensor([0.0, 0.0, 0.3])
    for n in (100_000, 1_000_000):
        xyz = room_scene(n, seed=n).cuda()
        model = V.BiasuttiVisibility(k=k, margin=margin, img_size=(W, H), r_max=30, r_min=0.5)
        _, _, xp, yp = V.camera_projection(xyz, cam, img_opk=opk, img_size=(W, H), r_max=30, r_min=0.5)
        s = search_set(xp, yp, W, margin)
        pos = torch.cat((s, torch.zeros((s.shape[0], 1), device=s.device)), 1)
        base = {"W": W, "H": H, "margin": margin, "k": k, "projected": int(xp.shape[0]), "search_set": int(s.shape[0]),
                "gpu": ident["name"], "power_limit_w": ident["power_limit_w"]}
        emit({"what": "knn_grid_image_plane", **base, **timed(lambda: knn_grid(pos, k), args.iters, args.warmup)})
        out = model(xyz, cam, img_opk=opk)
        emit({"what": "biasutti_call", **base, "kept": int(out["idx"].shape[0]),
              **timed(lambda: model(xyz, cam, img_opk=opk), args.iters, args.warmup)})
        if n == 100_000:
            q = s[:xp.shape[0]].contiguous()
            ref = dense_knn(q, s, k)
            got = knn_grid(pos, k)[:xp.shape[0]]
            # same k-th distance (the index order of ties and cdist's rounding may differ)
            dk = lambda nb: ((q - s[nb[:, -1]]) ** 2).sum(1)  # noqa: E731
            agree = float(((dk(ref) - dk(got)).abs() <= 1e-3 * dk(got).clamp_min(1e-6)).float().mean())
            emit({"what": "dense_cdist_topk", **base, "kth_distance_agreement": agree,
                  **timed(lambda: dense_knn(q, s, k), max(3, args.iters // 4), 1)})
        del xyz, s, pos, out
        torch.cuda.empty_cache()

    pos = cloud_300k().cuda()
    libs = [("this", _lib.load())]
    if args.baseline_lib:
        libs.append(("baseline", load_lib(args.baseline_lib)))
    res = {name: [] for name, _ in libs}
    for rnd in range(3):                                     # alternate the libraries
        for name, lib in libs:
            saved = _lib._loaded[_lib.B200.file]
            _lib._loaded[_lib.B200.file] = lib
            try:
                nb = knn_grid(pos, 20)
                r = timed(lambda: knn_grid(pos, 20), args.iters, args.warmup)
            finally:
                _lib._loaded[_lib.B200.file] = saved
            res[name].append((r, nb))
    ref_nb = res["this"][0][1]
    for name, runs in res.items():
        ms = sorted(r["median_ms"] for r, _ in runs)
        emit({"what": "knn_grid_cloud_k20", "library": name, "n": int(pos.shape[0]), "k": 20,
              "median_of_round_medians_ms": ms[1], "round_medians_ms": [r["median_ms"] for r, _ in runs],
              "identical_to_this": all(torch.equal(nb, ref_nb) for _, nb in runs),
              "gpu": ident["name"], "power_limit_w": ident["power_limit_w"]})
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for d in lines:
            f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
