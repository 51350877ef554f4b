#!/usr/bin/env python
"""Per-kernel measurements for the SURVEY.md section-8 rows other than the fused view attention
(which has bench.py and tools/bench_shapes.py): one JSON line per operator with its device time
(CUDA events, L2 flushed between iterations, median of K), the algorithmic bytes of the launch
and the fraction of the measured HBM peak -- or, for the atomic / latency-bound integer kernels,
the natural throughput unit (Mpoints/s, Mkeys/s).

    python tools/bench_rows.py [--only name,...] [--out FILE]

Shapes follow the S3DIS batch of SURVEY.md Appendix E (4 x 40 k-point spheres, ~8 views per point,
64-channel feature maps) scaled up where a launch would otherwise be too short to time.
Everything goes through the public operators (deepviewagg_b200.ops / core.multimodal), i.e. the C ABI.
"""
import argparse
import contextlib
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def peak_gbs():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0          # H100 SXM data sheet


class Timer:
    def __init__(self, dev, iters):
        self.flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        self.iters = iters

    def __call__(self, fn, warmup=2):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(self.iters):
            self.flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return statistics.median(ts)


@contextlib.contextmanager
def deterministic():
    """torch.use_deterministic_algorithms(True) without torch's NaN fill of torch.empty, so that a row
    times the library's kernels rather than the fill."""
    import torch.utils.deterministic as tud
    prev, fill = torch.are_deterministic_algorithms_enabled(), tud.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True)
    tud.fill_uninitialized_memory = False
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)
        tud.fill_uninitialized_memory = fill


def ragged_ptr(N, mean, dev, gen, p_empty=0.1):
    counts = torch.poisson(torch.full((N,), float(mean), device=dev), generator=gen).long()
    counts[torch.rand(N, device=dev, generator=gen) < p_empty] = 0
    return torch.cat([torch.zeros(1, dtype=torch.long, device=dev), counts.cumsum(0)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="")
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    from deepviewagg_b200 import ops, _lib
    from deepviewagg_b200.core.multimodal import visibility as vis
    from deepviewagg_b200.core.multimodal import csr as csrmod
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gen = torch.Generator(device=dev).manual_seed(7)
    T = Timer(dev, args.iters)
    peak = peak_gbs()
    only = set(filter(None, args.only.split(",")))
    lines = []
    from bench import gpu_identity
    ident = gpu_identity(0)            # read, not set: the card and power limit are part of every number
    print(json.dumps({"gpu": ident}), flush=True)

    def emit(name, row, ms, bytes_=None, units=None, unit_name=None, note=""):
        d = {"op": name, "survey_row": row, "ms": round(ms, 4), "gpu": ident["name"],
             "power_limit_w": ident["power_limit_w"]}
        if bytes_ is not None:
            gbs = bytes_ / (ms * 1e-3) / 1e9
            d.update({"algorithmic_bytes": int(bytes_), "gbs": round(gbs, 1), "frac_of_hbm_peak": round(gbs / peak, 3)})
        if units is not None:
            d.update({unit_name: round(units / (ms * 1e-3) / 1e6, 2)})
        if note:
            d["note"] = note
        print(json.dumps(d), flush=True)
        lines.append(d)

    def want(name):
        return not only or name in only

    # ---- P1 / T1 segment_csr (max) fwd + bwd, P8 gather_csr, P7 segment softmax ------------------
    N, C = 1_000_000, 64
    ptr = ragged_ptr(N, 8, dev, gen)
    V = int(ptr[-1])
    x = torch.randn(V, C, device=dev, generator=gen)
    if want("segment_csr_max"):
        xr = x.clone().requires_grad_(True)
        out = ops.segment_csr(xr, ptr, reduce="max")
        go = torch.randn_like(out)
        emit("segment_csr_max_fwd", "P1/T1", T(lambda: ops.segment_csr(x, ptr, reduce="max")),
             V * C * 4 + N * C * 4 + N * 8, note=f"[{V},{C}] f32 -> [{N},{C}], ~8 rows per segment")
        emit("segment_csr_max_bwd", "P1/T1", T(lambda: torch.autograd.grad(out, xr, go, retain_graph=True)),
             V * C * 4 + N * C * (4 + 8), note="zero-fill of grad_src included; arg table int64 [N,C]")
    if want("segment_csr_sum"):
        emit("segment_csr_sum_fwd", "P1/T1", T(lambda: ops.segment_csr(x, ptr, reduce="sum")),
             V * C * 4 + N * C * 4 + N * 8)
    if want("gather_csr"):
        pts = torch.randn(N, 32, device=dev, generator=gen)
        emit("gather_csr", "P8", T(lambda: ops.gather_csr(pts, ptr)), N * 32 * 4 + V * 32 * 4 + N * 8,
             note=f"[{N},32] -> [{V},32]")
    if want("segment_softmax"):
        sc = torch.randn(V, 4, device=dev, generator=gen)
        emit("segment_softmax_csr_fwd", "P7", T(lambda: ops.segment_softmax_csr(sc, ptr, scaling=True)),
             2 * V * 4 * 4 + N * 8, note=f"[{V},4] scores")
    del x

    # ---- P4 QK scores ----------------------------------------------------------------------------
    if want("qk_scores"):
        G, D = 4, 8
        K = torch.randn(V, G * D, device=dev, generator=gen, requires_grad=True)
        Q = torch.randn(N, G * D, device=dev, generator=gen, requires_grad=True)
        out = ops.qk_scores(K, Q, ptr, G)
        go = torch.randn_like(out)
        emit("qk_scores_fwd", "P4", T(lambda: ops.qk_scores(K, Q, ptr, G)),
             V * G * D * 4 + N * G * D * 4 + V * G * 4 + N * 8, note=f"K [{V},{G*D}], Q [{N},{G*D}]")
        emit("qk_scores_bwd", "P4", T(lambda: torch.autograd.grad(out, [K, Q], go, retain_graph=True)),
             2 * V * G * D * 4 + 2 * N * G * D * 4 + V * G * 4 + N * 8)
        del K, Q

    # ---- I5 + P1 fused feature-map gather + atomic pool -----------------------------------------
    if want("gather_pool"):
        B, Cm, H, W = 16, 64, 256, 512
        Pn = 1_200_000
        images = torch.randint(0, B, (Pn,), device=dev, generator=gen).sort().values
        pix = torch.stack([torch.randint(0, W, (Pn,), device=dev, generator=gen),
                           torch.randint(0, H, (Pn,), device=dev, generator=gen)], 1).to(torch.int16)
        aptr = torch.arange(Pn + 1, device=dev)       # exact splatting: one pixel per view
        for cl in (True, False):
            fm = torch.randn((B, H, W, Cm) if cl else (B, Cm, H, W), device=dev, generator=gen)
            fr = fm.clone().requires_grad_(True)
            out = ops.gather_pool(fr, images, pix, aptr, "max", channels_last=cl)
            go = torch.randn_like(out)
            tag = "nhwc" if cl else "nchw"
            emit(f"gather_pool_fwd_{tag}", "I5+P1",
                 T(lambda: ops.gather_pool(fm, images, pix, aptr, "max", channels_last=cl)),
                 Pn * Cm * 4 * 2 + Pn * (8 + 4 + 8 + 8),
                 note=f"{Pn} pixels from [{B},{Cm},{H},{W}] maps -> [{Pn},{Cm}]" +
                      ("" if cl else "; NCHW: every element is its own 32-byte sector"))
            emit(f"gather_pool_bwd_{tag}", "I5+P1",
                 T(lambda: torch.autograd.grad(out, fr, go, retain_graph=True)),
                 Pn * Cm * 4 * 3 + fm.numel() * 4 + Pn * (8 + 4 + 8 + 8),
                 note="grad_out read + read-modify-write of the touched map pixels + zero-fill of the "
                      "whole map gradient; fp32 reductions (16-byte red.v4 on the channels-last path)")
            with deterministic():
                emit(f"gather_pool_bwd_det_{tag}", "I5+P1",
                     T(lambda: torch.autograd.grad(out, fr, go, retain_graph=True)),
                     Pn * Cm * 4 + fm.numel() * 4 + Pn * (8 + 4 + 8 + 8),
                     note="torch.use_deterministic_algorithms(True): pixel-bucket index (counting sort) + "
                          "one ordered fp32 sum per map element, whole map gradient written once; "
                          "fill_uninitialized_memory=False" + ("" if cl else "; NCHW: scalar reducer"))
            del fm, fr, out
    if want("interp_pool"):
        # reuse-heavy: a mapping at 4x the map resolution, ~3 pixels per view, 4 bilinear corners per pixel
        B, Cm, H, W = 16, 64, 64, 128
        msz = (4 * W, 4 * H)
        Vn = 400_000
        iptr = ragged_ptr(Vn, 3, dev, gen, p_empty=0.0)
        Pn = int(iptr[-1])
        images = torch.randint(0, B, (Vn,), device=dev, generator=gen)
        pix = torch.stack([torch.randint(0, msz[0], (Pn,), device=dev, generator=gen),
                           torch.randint(0, msz[1], (Pn,), device=dev, generator=gen)], 1).to(torch.int16)
        fm = torch.randn((B, H, W, Cm), device=dev, generator=gen)
        fr = fm.clone().requires_grad_(True)
        out = ops.interp_pool(fr, images, pix, iptr, msz, reduce="max", channels_last=True)
        go = torch.randn_like(out)
        note = (f"{Pn} pixels at {msz[0]}x{msz[1]} -> {Vn} views (max) from [{B},{H},{W},{Cm}] maps, "
                f"~{4 * Pn // (B * H * W)} contributions per map pixel")
        emit("interp_pool_bwd_atomic_nhwc", "I5b+P1", T(lambda: torch.autograd.grad(out, fr, go, retain_graph=True)),
             Vn * Cm * 4 + fm.numel() * 4 * 3 + Vn * Cm * 8, note=note + "; zero-fill + red.v4 into the map")
        with deterministic():
            emit("interp_pool_bwd_det_nhwc", "I5b+P1",
                 T(lambda: torch.autograd.grad(out, fr, go, retain_graph=True)),
                 Vn * Cm * 4 + fm.numel() * 4 + Vn * Cm * 8,
                 note=note + "; deterministic: bucket index + ordered sums; fill_uninitialized_memory=False")
        del fm, fr, out

    # ---- P9 BN + LeakyReLU ------------------------------------------------------------------------
    if want("bn_act"):
        R, Cb = 8_000_000, 32
        z = torch.randn(R, Cb, device=dev, generator=gen)
        bn = torch.nn.BatchNorm1d(Cb).to(dev).train()
        zr = z.clone().requires_grad_(True)
        y = ops.batch_norm_act(zr, bn, 0.2)
        go = torch.randn_like(y)
        emit("bn_lrelu_fwd", "P9", T(lambda: ops.batch_norm_act(z, bn, 0.2)), 3 * R * Cb * 4,
             note=f"[{R},{Cb}] train mode: stats pass + apply pass")
        emit("bn_lrelu_bwd", "P9", T(lambda: torch.autograd.grad(y, zr, go, retain_graph=True)), 5 * R * Cb * 4)
        del z, zr, y, go

    # ---- Z1-Z3 projection + splat boxes + z-buffer ------------------------------------------------
    if want("visibility"):
        n = 1_000_000
        xyz = (torch.rand(n, 3, device=dev, generator=gen) - 0.5) * torch.tensor([20.0, 20.0, 4.0], device=dev)
        cam = torch.zeros(3, device=dev)
        opk = torch.zeros(3, device=dev)
        kw = dict(img_size=(2048, 1024), crop_top=0, crop_bottom=0, r_max=30.0, r_min=0.5)

        def proj():
            return vis.camera_projection(xyz, cam, img_opk=opk, camera="s3dis_equirectangular", **kw)
        idx, dist, xp, yp = proj()
        emit("camera_projection_equirect", "Z1", T(proj), units=n, unit_name="mpoints_per_s",
             note=f"{n} points -> {idx.numel()} inside; includes the nonzero() compaction")
        for exact in (False, True):
            def zb():
                return vis.visibility_from_splatting(xp, yp, dist, img_size=(2048, 1024), voxel=0.03, k_swell=1.0,
                                                     d_swell=1000, exact=exact, camera="s3dis_equirectangular")
            r = zb()
            emit(f"splat_zbuffer_exact{int(exact)}", "Z2+Z3", T(zb), units=idx.numel(), unit_name="mpoints_per_s",
                 note=f"{idx.numel()} points splatted into 2048x1024, {r[0].numel()} visible pixels; "
                      "boxes + 64-bit atomicMin raster + resolve + nonzero()")

    # ---- C1 CSR pointers / selection -------------------------------------------------------------
    if want("csr"):
        n_ids, groups = 16_000_000, 2_000_000
        ids = torch.randint(0, groups, (n_ids,), device=dev, generator=gen).sort().values
        emit("csr_pointers_from_sorted", "C1", T(lambda: csrmod.pointers_from_sorted(ids, groups)),
             n_ids * 8 + groups * 8, units=n_ids, unit_name="mkeys_per_s")
        p = csrmod.pointers_from_sorted(ids, groups)
        sel = torch.randperm(groups, device=dev, generator=gen)[: groups // 2]
        emit("csr_select_values", "C1", T(lambda: csrmod.select_values(p, sel)), units=sel.numel(),
             unit_name="mgroups_per_s", note="new pointers + value index for a random half of the groups")

    # ---- I1 / I4 mapping re-indexing on the device (native counting sort + warp rank sort, csrc/mapping_build.cu) ----
    if want("mapping"):
        from deepviewagg_b200.core.multimodal.image import ImageMapping
        npts, nimg = 400_000, 64
        m = 3_000_000
        pid = torch.randint(0, npts, (m,), device=dev, generator=gen)
        iid = torch.randint(0, nimg, (m,), device=dev, generator=gen)
        pixs = torch.stack([torch.randint(0, 1024, (m,), device=dev, generator=gen),
                            torch.randint(0, 512, (m,), device=dev, generator=gen)], 1)
        feats = torch.rand(m, 8, device=dev, generator=gen)

        def build():
            return ImageMapping.from_dense(pid, iid, pixs, feats, num_points=npts)
        mp = build()
        emit("image_mapping_from_dense", "I1", T(build), units=m, unit_name="mtriples_per_s",
             note=f"{m} (point,image,pixel) triples, {npts} points, {nimg} images")
        vox = torch.randint(0, npts // 4, (npts,), device=dev, generator=gen)
        vox[: npts // 4] = torch.arange(npts // 4, device=dev)          # every output voxel present (image.py:2220)
        emit("select_points_merge", "I4", T(lambda: mp.select_points(vox, mode="merge")), units=m,
             unit_name="mtriples_per_s", note="4:1 voxel merge (strided sparse conv re-indexing)")

    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")
    assert _lib.launch_count() > 0


if __name__ == "__main__":
    main()
