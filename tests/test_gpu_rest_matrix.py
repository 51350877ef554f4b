"""Every kernel of tests/test_rest_matrix_table.py launched and proven launched: each scenario runs once under the
kernel recorder of tests/test_gpu_kernel_matrix.py and checks its results against the references and bounds of the
table's module docstring; each case asserts, by name, that its kernel ran in its scenario."""
import contextlib
import functools

import numpy as np
import pytest
import torch

from oracle import color_oracle as CO
from oracle import deterministic_oracle as DO
from oracle import image_resample_oracle as IR
from oracle import visibility_oracle as VO
from oracle.neighborhood_oracle import knn_bruteforce, neighborhood_features
from oracle.no3d_oracle import knn_query_bruteforce
from test_gpu_kernel_matrix import place, record
from test_kernel_matrix_table import CPP, DTYPES, TINY, U_S, V16, kname, va_bounds, va_inputs, va_reference, violations
from test_rest_matrix_table import (CASE_IDS, CASES, SCAN_CARRY_BUCKETS, TABLE, canonical, mapping_feature_bound,
                                    nll_bounds, nll_reference)

pytestmark = pytest.mark.gpu
SEEN = set()
WANT = {}
for _c in CASES:
    WANT.setdefault(_c["scenario"], set()).add(_c["kernel"])


@contextlib.contextmanager
def deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


# ------------------------------------------------------------------------------------------------
# k-NN: clouds near the origin and translated far from it, with a cell size of a few cm
# ------------------------------------------------------------------------------------------------
KNN_SHIFTS = (0.0, 1e3, 1e4, 1e5)


def _cloud(seed, shift):
    """3000 points in a 1 m x 1 m x 0.1 m slab (duplicates, a planar patch at z = 0 near the origin), one isolated
    point 30 m away, all translated by `shift` on x and y and shift / 10 on z, then rounded to fp32."""
    rng = np.random.default_rng(seed)
    p = rng.random((3000, 3)) * np.array([1.0, 1.0, 0.1])
    p[1::40] = p[0::40][:p[1::40].shape[0]]                      # duplicated points: d2 = 0, ties by index
    p[2000:2400, 2] = 0.0                                         # planar patch
    p[-1] = (30.0, 1.0, 0.05)                                     # isolated: the self case's exhaustive fallback
    return (p + np.array([shift, shift, shift / 10])).astype(np.float32)


def _knn_self(kmax):
    from deepviewagg_b200.core.multimodal.mapping import knn_grid
    ks = (1, 20, 64) if kmax == 64 else (65, 128)
    for shift in KNN_SHIFTS:
        p = _cloud(7, shift)
        for k in ks:
            nbr, d2 = knn_grid(torch.from_numpy(p).cuda(), k, cell_size=0.05, return_dist2=True)
            want_n, want_d = knn_bruteforce(p, k)
            bad = np.nonzero((nbr.cpu().numpy() != want_n).any(1) | (d2.cpu().numpy() != want_d).any(1))[0]
            assert bad.size == 0, f"knn_grid shift={shift} k={k}: {bad.size} rows differ, first {bad[:5]}"


def _knn_query(kmax):
    from deepviewagg_b200.core.multimodal.mapping import knn_query
    ks = (1, 64) if kmax == 64 else (65, 128)
    for shift in KNN_SHIFTS:
        s = _cloud(8, shift)[:-1]
        rng = np.random.default_rng(9)
        q = np.concatenate([rng.random((2000, 3)) * np.array([1.4, 1.4, 0.3]) - np.array([0.2, 0.2, 0.1]),
                            rng.random((200, 3)) + np.array([5.0, 0.0, 0.0])])       # outside the grid: coarse
        q = (q + np.array([shift, shift, shift / 10])).astype(np.float32)
        q[:50] = s[:50]                                                             # queries on search points
        for k in ks:
            nbr, d2 = knn_query(torch.from_numpy(q).cuda(), torch.from_numpy(s).cuda(), k, cell_size=0.05,
                                return_dist2=True)
            want_n, want_d = knn_query_bruteforce(q, s, k)
            bad = np.nonzero((nbr.cpu().numpy() != want_n).any(1) | (d2.cpu().numpy() != want_d).any(1))[0]
            assert bad.size == 0, f"knn_query shift={shift} k={k}: {bad.size} rows differ, first {bad[:5]}"


def _nbr_features():
    from conftest import load_golden
    from deepviewagg_b200.core.multimodal.image import ImageMapping, SameSettingImageData
    from deepviewagg_b200.core.multimodal.mapping import NeighborhoodBasedMappingFeatures
    g = load_golden("neighborhood_features")                     # holds a duplicated point: d2 = 0, inf density
    W, H, n_img = [int(v) for v in g["size"]]
    pos = g["pos"].numpy()
    nbr, _ = knn_bruteforce(pos, 20)
    infinite = False
    for kw in (dict(k=[20, 5, 5], voxel=0.05), dict(k=[7, 3], density=False), dict(k=16, occlusion=False),
               dict(k=[2, 1], occlusion=False)):                 # k = 1: the point itself, d2 = 0
        im = SameSettingImageData(pos=torch.zeros(n_img, 3), opk=torch.zeros(n_img, 3), ref_size=(W, H),
                                  proj_upscale=1, downscale=1)
        im.mappings = ImageMapping.from_dense(g["pid"], g["iid"], g["pix"], None, num_points=pos.shape[0])
        im = im.to("cuda")
        klist = kw["k"] if isinstance(kw["k"], list) else [kw["k"]]
        kn = nbr[:, :max(klist)]                                  # the transform takes [N, max k] neighbours
        out = NeighborhoodBasedMappingFeatures(**kw)(g["pos"], im, neighbors=torch.from_numpy(kn).cuda())
        want = neighborhood_features(pos, kn, im.mappings.pointers.cpu().numpy(), im.mappings.images.cpu().numpy(),
                                     klist, voxel=kw.get("voxel", 1), density=kw.get("density", True),
                                     occlusion=kw.get("occlusion", True))
        got = out.mappings.features.cpu().numpy()
        assert np.array_equal(got, want, equal_nan=True), kw
        infinite |= bool(np.isinf(want).any())
    assert infinite


# ------------------------------------------------------------------------------------------------
# mapping build, view_cat_sorting, CSR bookkeeping
# ------------------------------------------------------------------------------------------------
PIX_T = {"i16": torch.int16, "i32": torch.int32, "i64": torch.int64}


def _mapping_inputs(px, n_points, n_items, seed):
    """Random items plus buckets (items of one point) of exactly 1, 32, 33 and 1200 items, every item of a bucket on
    the same image (the rank sort orders by pixel, ties by item); points 0, 2-4, 6, 8 and the last 3 unseen."""
    rng = np.random.default_rng(seed)
    pid = rng.integers(10, n_points - 3, n_items)
    iid = rng.integers(0, 7, n_items)
    pos = rng.permutation(n_items)
    for p, L in ((1, 1), (5, 1200), (7, 32), (9, 33)):
        sel, pos = pos[:L], pos[L:]
        pid[sel], iid[sel] = p, 3
    hi = {"i16": 60, "i32": 40000, "i64": 65000}[px]
    pix = rng.integers(0, hi, (n_items, 2))
    pix[1::3] = pix[0::3][:pix[1::3].shape[0]]                    # duplicated (point, image, pixel) items
    return pid, iid, pix


def _check_mapping(px, n_points, n_items, seed, F=(16, 1, None)):
    from deepviewagg_b200.core.multimodal.image import ImageMapping
    pid, iid, pix = _mapping_inputs(px, n_points, n_items, seed)
    rng = np.random.default_rng(seed + 1)
    for f in F:
        feat = None if f is None else rng.random((n_items, f)).astype(np.float32)
        got = ImageMapping.from_dense(torch.from_numpy(pid).cuda(), torch.from_numpy(iid).cuda(),
                                      torch.from_numpy(pix).to(PIX_T[px]).cuda(),
                                      None if feat is None else torch.from_numpy(feat).cuda(), num_points=n_points)
        ref = VO.image_mapping_from_dense(pid, iid, pix, None, n_points)
        assert np.array_equal(got.pointers.cpu().numpy(), ref["pointers"])
        assert np.array_equal(got.images.cpu().numpy(), ref["images"])
        ap = ref["atomic_pointers"]
        assert np.array_equal(got.values[1].pointers.cpu().numpy(), ap)
        assert got.pixels.dtype == PIX_T[px] and np.array_equal(got.pixels.cpu().numpy().astype(np.int64), ref["pixels"])
        if feat is not None:
            fs = feat[VO.lexargsort(pid, iid)]
            mean = np.add.reduceat(fs.astype(np.float64), ap[:-1], axis=0) / np.diff(ap)[:, None]
            err = np.abs(got.features.cpu().numpy().astype(np.float64) - mean)
            assert (err <= mapping_feature_bound(fs, ap, mean)).all(), f"features F={f}"
    # ids outside [0, num_points) are rejected
    with pytest.raises(IndexError):
        ImageMapping.from_dense(torch.from_numpy(pid).cuda() + n_points, torch.from_numpy(iid).cuda(),
                                torch.from_numpy(pix).to(PIX_T[px]).cuda(), None, num_points=n_points)


def _view_cat():
    from deepviewagg_b200.core.multimodal.image import ImageData, ImageMapping, SameSettingImageData
    rng = np.random.default_rng(12)
    N, ims, dense = 20000, [], []
    for s, (n_img, n_items) in enumerate(((4, 90000), (2, 30000), (3, 1), (5, 150000))):
        pid, iid = rng.integers(0, N, n_items), rng.integers(0, n_img, n_items)
        pix = rng.integers(0, 32, (n_items, 2)).astype(np.int16)
        im = SameSettingImageData(pos=torch.zeros(n_img, 3), opk=torch.zeros(n_img, 3), ref_size=(32 + s, 32),
                                  proj_upscale=1, downscale=1)
        im.mappings = ImageMapping.from_dense(torch.from_numpy(pid), torch.from_numpy(iid), torch.from_numpy(pix),
                                              None, num_points=N)
        ims.append(im)
        ref = VO.image_mapping_from_dense(pid, iid, pix, None, N)
        dense.append(np.repeat(np.arange(N), np.diff(ref["pointers"])))
    gpu = ImageData(ims).to("cuda")
    srt, csr = gpu._view_cat_native()
    allv = np.concatenate(dense)
    assert np.array_equal(srt.cpu().numpy(), np.argsort(allv, kind="stable"))
    assert np.array_equal(csr.cpu().numpy(), np.concatenate([[0], np.cumsum(np.bincount(allv, minlength=N))]))


def _csr_build():
    from deepviewagg_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(1)
    for n, ng in ((0, 5), (1, 1), (5000, 700), (100000, 100000), (10, 1000)):
        ids = np.sort(rng.integers(0, ng, n)).astype(np.int64)
        ref = VO.pointers_from_sorted_with_empties(ids, ng) if n else np.zeros(ng + 1, np.int64)
        d_ids = torch.from_numpy(ids).cuda()
        ptr = torch.full((ng + 1,), -7, dtype=torch.int64, device="cuda")
        _lib.check(lib.dva_csr_pointers_from_sorted(_lib.ptr(d_ids), _lib.ptr(ptr), n, ng, _lib.stream_ptr()), "csr")
        assert np.array_equal(ptr.cpu().numpy(), ref), (n, ng)
    counts = rng.integers(0, 5, 3000)
    counts[::7] = 0
    pointers = np.concatenate([[0], np.cumsum(counts)])
    sel = rng.integers(0, 3000, 1200)
    pn_ref, val_ref = VO.index_select_pointers(pointers, sel)
    val = torch.empty(int(pn_ref[-1]), dtype=torch.int64, device="cuda")
    d_ptr, d_sel, d_pn = (torch.from_numpy(a).cuda() for a in (pointers, sel, pn_ref))
    _lib.check(lib.dva_csr_select_values(_lib.ptr(d_ptr), _lib.ptr(d_sel), _lib.ptr(d_pn), _lib.ptr(val), sel.size,
                                         val.numel(), _lib.stream_ptr()), "select")
    assert np.array_equal(val.cpu().numpy(), val_ref)


# ------------------------------------------------------------------------------------------------
# bucket-index users: deterministic pool and row scatter, coverage index
# ------------------------------------------------------------------------------------------------
def _det_pool(B, H, W, C, Vw, seed, pix_types=(torch.int16, torch.int32), interps=(False, True)):
    from test_gpu_deterministic import _mapping, _oracle, _run
    gen = torch.Generator().manual_seed(seed)
    for interp in interps:
        msz = (2 * W + 3, 2 * H + 1) if interp else None
        img, pix, aptr = _mapping(gen, B, H, W, Vw, msz or (W, H), oob=not interp)
        fmap = torch.randn(B, C, H, W, generator=gen)
        go = torch.randn(Vw, C, generator=gen)
        for pdt in pix_types:
            for red in ("sum", "max"):
                with deterministic():
                    got = _run(fmap, torch.float32, False, img, pix.to(pdt), aptr, red, msz, go)
                assert torch.equal(got, _oracle(fmap, torch.float32, img, pix, aptr, red, msz, go)), (interp, pdt, red)


def _det_rows(dt, R, V, widths, seed):
    from deepviewagg_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    for C, off in widths:
        src = torch.randn(V, C, generator=gen).to(DTYPES[dt])
        idx = torch.randint(0, R, (V,), generator=gen)
        idx[::17] = R                                              # outside [0, R): skipped
        idx[::19] = -1
        idx[: min(V, 2000)] = 3                                    # one row fed 2000 times
        with deterministic():
            got = ops._scatter_add_rows(place(src, off), idx.cuda(), R).cpu()
        want = DO.scatter_add_rows_ordered(src.float().numpy(), idx.numpy(), R)
        assert torch.equal(got, torch.from_numpy(want)), (dt, C, off)


def _coverage_big():
    """2.5 M points (buckets of the point index), 40 images; the unseen counts after every pick against numpy."""
    from deepviewagg_b200 import ops
    rng = np.random.default_rng(3)
    N, n_img = 2_500_000, 40
    gimg, vpoint = [], []
    for i in range(n_img):
        pts = np.unique(rng.integers(0, N, int(rng.integers(10_000, 120_000))))
        gimg.append(np.full(pts.size, i))
        vpoint.append(pts)
    gimg, vpoint = np.concatenate(gimg), np.concatenate(vpoint)
    cov = ops.CoverageIndex(torch.from_numpy(gimg).cuda(), torch.from_numpy(vpoint).cuda(), n_img, N)
    unseen = np.bincount(gimg, minlength=n_img).astype(np.int64)
    seen = np.zeros(N, dtype=bool)
    assert np.array_equal(cov.unseen.cpu().numpy(), unseen)
    for g in (5, 17, 0, 39, 17):
        pts = vpoint[gimg == g]
        new = pts[~seen[pts]]
        seen[new] = True
        hit = np.zeros(N, dtype=bool)
        hit[new] = True
        unseen -= np.bincount(gimg[hit[vpoint]], minlength=n_img)
        cov.pick(g)
        assert np.array_equal(cov.unseen.cpu().numpy(), unseen), g


def _coverage():
    from test_transforms import check_memory_credit
    check_memory_credit("cuda")


# ------------------------------------------------------------------------------------------------
# segment / view-attention leftovers
# ------------------------------------------------------------------------------------------------
def _heuristic_arg():
    from deepviewagg_b200 import ops
    from oracle import pooling_oracle as O
    gen = torch.Generator().manual_seed(41)
    counts = torch.randint(0, 6, (700,), generator=gen)
    counts[::9] = 0
    ptr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)])
    V = int(ptr[-1])
    xmap = torch.randn(V, 3, generator=gen)
    xmap[1::4, 1] = xmap[0::4, 1][:xmap[1::4].shape[0]]            # ties in the picked feature: the first row wins
    x = torch.randn(V, 16, generator=gen)
    for mode in ("max", "min"):
        got = ops.heuristic_pool(x.cuda(), xmap.cuda(), ptr.cuda(), 1, mode=mode)
        assert torch.equal(got.cpu().double(), O.heuristic_pool(x.double(), xmap.double(), ptr, feat=1, mode=mode))


def _gate_reduce():
    from deepviewagg_b200 import ops
    inp = va_inputs(dict(dtype="f32", C=64, G=4), 0)
    ref = va_reference(inp)
    bnd = va_bounds(inp, ref)
    x = inp["x"].cuda().requires_grad_(True)
    c = inp["compat"].cuda().requires_grad_(True)
    gw, gb = inp["gw"].cuda().requires_grad_(True), inp["gb"].cuda().requires_grad_(True)
    out, _, _ = ops.view_attention(x, c, inp["ptr"].cuda(), inp["G"], gate_weight=gw, gate_bias=gb,
                                   group_scaling=inp["scaling"])
    ggw, ggb = torch.autograd.grad(out, [gw, gb], inp["gout"].cuda())
    for what, got in (("gw", ggw), ("gb", ggb)):
        n, msg = violations(got, ref[what], bnd[what])
        assert n == 0, f"grad {what}: {msg}"


# ------------------------------------------------------------------------------------------------
# projection, splat boxes, z-buffer
# ------------------------------------------------------------------------------------------------
def _zbuffer_random():
    from deepviewagg_b200.core.multimodal import visibility as V
    rng = np.random.default_rng(0)
    m, W, H = 200_000, 512, 256
    xp, yp = rng.uniform(0, W, m), rng.uniform(0, H, m)
    xp[::101], yp[::103] = 0.0, H - 1e-9                          # boxes clamped at the borders
    xp[::107] = W - 1e-9
    dist = rng.uniform(0.6, 20, m).astype(np.float32)
    tie = np.arange(0, m - 7, 7)
    dist[tie] = dist[tie + 3]                                     # equal distances: the lower index wins
    xp[tie], yp[tie] = xp[tie + 3], yp[tie + 3]
    for ct, cb in ((0, 0), (8, 8), (30, 0)):
        sp = VO.splat_boxes(xp, yp, dist, W, H, ct, cb, voxel=0.05)
        sg = V.splat_boxes(torch.from_numpy(xp).cuda(), torch.from_numpy(yp).cuda(), torch.from_numpy(dist).cuda(),
                           None, (W, H), ct, cb, voxel=0.05)
        assert np.array_equal(sg.cpu().numpy(), sp), (ct, cb)
        for exact in (False, True):
            i_ref, x_ref, y_ref, _ = VO.zbuffer(sp, dist, xp, yp, W, H, ct, cb, exact=exact)
            i2, x2, y2 = V.visibility_from_splatting(torch.from_numpy(xp).cuda(), torch.from_numpy(yp).cuda(),
                                                     torch.from_numpy(dist).cuda(), None, img_size=(W, H),
                                                     crop_top=ct, crop_bottom=cb, voxel=0.05, exact=exact)
            assert np.array_equal(i2.cpu().numpy(), i_ref) and np.array_equal(x2.cpu().numpy(), x_ref)
            assert np.array_equal(y2.cpu().numpy(), y_ref), (ct, cb, exact)


def _zbuffer_equirect():
    from test_gpu_integer import test_visibility_pipeline_vs_numba_fixture
    test_visibility_pipeline_vs_numba_fixture("crop")
    test_visibility_pipeline_vs_numba_fixture("nocrop")


def _zbuffer_camera():
    from test_gpu_integer import test_pinhole_fisheye_cameras_vs_numba_fixture
    test_pinhole_fisheye_cameras_vs_numba_fixture("kitti360_fisheye")
    test_pinhole_fisheye_cameras_vs_numba_fixture("scannet")


# ------------------------------------------------------------------------------------------------
# NLL
# ------------------------------------------------------------------------------------------------
def _nll_inputs(N, K, dt, with_csr, seed, minus_inf=True):
    gen = torch.Generator().manual_seed(seed)
    counts = torch.randint(0, 5, (N,), generator=gen)
    csr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)]) if with_csr else None
    V = int(csr[-1]) if with_csr else N
    x = 3 * torch.randn(V, K, generator=gen)
    x[::11] += 40                                                 # max-centring matters
    if minus_inf and K > 1:
        x[::3, 0] = -float("inf")                                 # the first logit -inf
        x[1::5, : K // 2] = -float("inf")                         # a -inf prefix
    lab = torch.randint(0, K, (N,), generator=gen)
    lab[torch.rand(N, generator=gen) < 0.2] = -1
    rows = torch.repeat_interleave(lab, counts) if with_csr else lab
    xs = x.to(DTYPES[dt])
    # a -inf at the target gives an infinite loss, as in torch: keep the targets finite here
    ok = rows >= 0
    xs[ok, rows[ok]] = x[ok, rows[ok]].clamp(min=-30).to(DTYPES[dt])
    return xs, lab, csr


def check_nll(x, lab, csr, dt):
    from deepviewagg_b200 import ops
    K = x.shape[1]
    xg = x.cuda().requires_grad_(True)
    loss = ops.csr_nll_loss(xg, lab.cuda(), None if csr is None else csr.cuda())
    g, = torch.autograd.grad(loss, xg)
    ref = nll_reference(x, lab, csr)
    b_loss, b_grad = nll_bounds(ref, K, dt)
    assert abs(float(loss) - float(ref["loss"])) <= b_loss, (float(loss), float(ref["loss"]), b_loss)
    n, msg = violations(g, ref["grad"], b_grad)
    assert n == 0, f"nll gradient: {msg}"


def _nll(dt):
    for K in (1, 13, 64):
        for with_csr in (True, False):
            check_nll(*_nll_inputs(2000, K, dt, with_csr, seed=K + with_csr), dt)


def _nll_edges():
    from deepviewagg_b200 import ops
    x, lab, csr = _nll_inputs(300, 13, "f32", True, seed=3)
    bad = lab.clone()
    bad[int(torch.nonzero(csr[1:] > csr[:-1])[0])] = 13           # out of range: stats[1]
    with pytest.raises(ValueError, match="label"):
        ops.csr_nll_loss(x.cuda(), bad.cuda(), csr.cuda())
    short = csr.clone()
    short[-1] -= 1                                                # csr does not span [0, V): stats[2]
    with pytest.raises(ValueError, match="csr_idx"):
        ops.csr_nll_loss(x.cuda(), lab.cuda(), short.cuda())
    none = torch.full_like(lab, -1)                               # count = 0: NaN, zero gradient
    xg = x.cuda().requires_grad_(True)
    loss = ops.csr_nll_loss(xg, none.cuda(), csr.cuda())
    assert torch.isnan(loss) and (torch.autograd.grad(loss, xg)[0] == 0).all()
    # points without views
    lab2 = torch.cat([lab, torch.tensor([2, 4])])
    check_nll(x, lab2, torch.cat([csr, csr[-1:], csr[-1:]]), "f32")


# ------------------------------------------------------------------------------------------------
# image kernels
# ------------------------------------------------------------------------------------------------
def _image_stats(px):
    from test_gpu_transforms import test_mapping_image_stats_against_scatter_reduce
    test_mapping_image_stats_against_scatter_reduce(PIX_T[px])


def _center_roll():
    from test_transforms import check_quantisation
    check_quantisation("cuda")


def _remap():
    from test_gpu_transforms import test_image_remap_against_torch
    test_image_remap_against_torch(torch.uint8, True)


def _resample(C):
    from deepviewagg_b200 import ops
    rng = np.random.default_rng(C)
    imgs = rng.integers(0, 256, (3, 41, 57, C), dtype=np.uint8)
    imgs[..., C - 1] = 255 - imgs[..., 0]                         # the last channel differs from every other
    for size, box in (((23, 17), None), ((80, 60), (3.5, 2.25, 50.75, 40.5)), ((57, 20), None), ((30, 41), None)):
        out = ops.image_resample(torch.from_numpy(imgs).cuda().permute(0, 3, 1, 2), size, boxes=box)
        ref = np.stack([IR.resize(a, size, box) for a in imgs]).transpose(0, 3, 1, 2)
        assert np.array_equal(out.cpu().numpy(), ref), (C, size, box)


def _nonstatic(C):
    from deepviewagg_b200 import ops
    g = torch.Generator().manual_seed(3 + C)
    imgs = torch.randint(0, 3, (5, C, 37, 53), generator=g, dtype=torch.uint8)
    ref = (imgs[1:] != imgs[:1]).all(dim=1).any(dim=0).t()
    got = ops.nonstatic_mask(imgs.cuda())
    assert torch.equal(got.cpu(), ref), C


def _to_float(tag, vec):
    from deepviewagg_b200 import ops
    g = torch.Generator().manual_seed(5)
    for C in (1, 3, 4):
        shape = (2, C, 16, 32) if vec else (2, C, 9, 13)          # HW % 16 != 0 on the scalar path
        x = torch.randint(0, 256, shape, dtype=torch.uint8, generator=g)
        if tag == "u8":
            src, want = x, CO.to_float(x.numpy())
            mean = std = None
        else:
            src = torch.from_numpy(CO.to_float(x.numpy()))
            mean, std = [0.1, 0.2, 0.3, 0.4][:C], [0.3, 0.25, 0.5, 0.7][:C]
            want = np.stack([CO.normalize(a, mean, std) for a in src.numpy()])
        xg = place(src, 0 if vec else 1)                          # the scalar path: also an odd storage offset
        got = ops.image_to_float(xg, mean, std) if mean else ops.image_to_float(xg)
        assert np.array_equal(got.cpu().numpy(), want), (tag, vec, C)


def _jitter():
    from deepviewagg_b200 import ops
    x = CO.color_input("ramps", 3, 19, 37)                        # HW % 16 != 0
    seq = [("brightness", 1.2), ("contrast", 0.7), ("saturation", 1.5)]
    want, _ = CO.color_jitter(x, [0, 1, 2, 3], (1.2, 0.7, 1.5))
    for off in (0, 1):                                            # 1: not 16-byte aligned
        got = ops.color_jitter_u8(place(torch.from_numpy(x), off), seq)
        assert np.array_equal(got.cpu().numpy(), want), off
    for fmt in (torch.contiguous_format, torch.channels_last):
        got = ops.color_jitter_u8(torch.from_numpy(x).cuda().contiguous(memory_format=fmt), seq)
        assert np.array_equal(got.cpu().numpy(), want), fmt


SCENARIO_FNS = {
    "knn_self64": lambda: _knn_self(64), "knn_self128": lambda: _knn_self(128),
    "knn_query64": lambda: _knn_query(64), "knn_query128": lambda: _knn_query(128),
    "nbr_features": _nbr_features,
    "mapping_i16": lambda: _check_mapping("i16", 5000, 60000, 1),
    "mapping_i32": lambda: _check_mapping("i32", 300, 40000, 2),
    "mapping_i64": lambda: _check_mapping("i64", 2000, 30000, 3),
    "mapping_big": lambda: _check_mapping("i16", 2_500_000, 3_000_000, 4, F=(None,)),
    "view_cat": _view_cat, "csr_build": _csr_build,
    "det_pool": lambda: _det_pool(3, 19, 23, 8, 3000, 1),
    # B H W = 2 x 1100 x 1100 = 2.42 M feature-map pixels: more buckets than one pass of the scan of block sums
    "det_pool_big": lambda: _det_pool(2, 1100, 1100, 4, 400_000, 2, pix_types=(torch.int32,), interps=(False,)),
    "det_rows_big": lambda: _det_rows("f32", 2_500_000, 3_000_000, ((4, 0),), 7),
    "coverage": _coverage, "coverage_big": _coverage_big,
    "heuristic_arg": _heuristic_arg, "gate_reduce": _gate_reduce,
    "zbuffer_random": _zbuffer_random, "zbuffer_equirect": _zbuffer_equirect, "zbuffer_camera": _zbuffer_camera,
    "nll_edges": _nll_edges,
    "center_roll": _center_roll, "remap": _remap, "jitter": _jitter,
}
for _dt in DTYPES:
    # VEC: 16-byte chunks of aligned rows; scalar: odd widths, or rows one element off 16-byte alignment
    SCENARIO_FNS[f"det_rows_{_dt}"] = functools.partial(_det_rows, _dt, 300, 5000,
                                                        ((8 * V16[_dt], 0), (13, 0), (2 * V16[_dt], 1)), 5)
    SCENARIO_FNS[f"nll_{_dt}"] = functools.partial(_nll, _dt)
for _px in PIX_T:
    SCENARIO_FNS[f"image_stats_{_px}"] = functools.partial(_image_stats, _px)
for _C in (1, 2, 3, 4):
    SCENARIO_FNS[f"resample_C{_C}"] = functools.partial(_resample, _C)
    SCENARIO_FNS[f"nonstatic_C{_C}"] = functools.partial(_nonstatic, _C)
for _tag in ("u8", "f32"):
    SCENARIO_FNS[f"to_float_{_tag}_vec"] = functools.partial(_to_float, _tag, True)
    SCENARIO_FNS[f"to_float_{_tag}_scalar"] = functools.partial(_to_float, _tag, False)

_RESULTS = {}


def run_scenario(name):
    """Run a scenario once per session under the recorder; its checks raise on a wrong result."""
    if name not in _RESULTS:
        try:
            _, names = record(SCENARIO_FNS[name], tuple(WANT[name]), canon=canonical, seen=SEEN)
            _RESULTS[name] = (names, None)
        except AssertionError as e:
            _RESULTS[name] = (set(), e)
    names, err = _RESULTS[name]
    if err is not None:
        raise err
    return names


def test_every_scenario_has_a_function():
    assert set(WANT) <= set(SCENARIO_FNS), sorted(set(WANT) - set(SCENARIO_FNS))


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_kernel(case):
    names = run_scenario(case["scenario"])
    assert case["kernel"] in names, f"{case['kernel']} did not run in {case['scenario']}; recorded: {sorted(names)}"


def test_large_cases_pass_the_scan_carry():
    """The large cases of every bucket-index user hold more buckets than one pass of bk::scan_of_sums."""
    assert 2_500_000 > SCAN_CARRY_BUCKETS and 2 * 1100 * 1100 > SCAN_CARRY_BUCKETS


def test_nll_row_with_a_leading_minus_inf():
    """A row whose first logit is -inf: finite loss and gradient, as log_softmax + nll_loss in float64."""
    x = torch.tensor([[-float("inf"), 1.0, 2.0], [-float("inf"), -float("inf"), 0.5], [0.0, -float("inf"), 3.0]])
    lab = torch.tensor([1, 2, 0])
    from deepviewagg_b200 import ops
    for dt in DTYPES:
        xg = x.to(DTYPES[dt]).cuda().requires_grad_(True)
        loss = ops.csr_nll_loss(xg, lab.cuda())
        g, = torch.autograd.grad(loss, xg)
        assert torch.isfinite(loss) and torch.isfinite(g).all(), (dt, float(loss), g)
        check_nll(x.to(DTYPES[dt]), lab, None, dt)


def test_every_kernel_launched():
    """The union of the kernels recorded by all scenarios is exactly the table (scenarios not run yet in this
    session, e.g. under -k, are run here)."""
    for name in WANT:
        try:
            run_scenario(name)
        except AssertionError:
            pass
    table = set(TABLE)
    assert SEEN == table, {"never launched": sorted(table - SEEN), "launched without a case": sorted(SEEN - table)}
