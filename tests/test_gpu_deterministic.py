"""Deterministic backwards under torch.use_deterministic_algorithms(True): the feature-map gradients of
gather_pool / interp_pool / sparse_interpolation_pixels and the rows scatter-add of view_attention are
bit-identical to the ordered CPU oracle (oracle/deterministic_oracle.py), agree with the atomic path,
and a training step of the branch gives the same gradients twice."""
import contextlib

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import deterministic_oracle as D

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


# layout -> (channels, channels_last, number of views): "nchw" gathers few pixels (direct NCHW
# kernels), "nchw_t" enough to be transposed to channels-last; cl8 / cl64 / cl160: 16-byte chunks;
# cl12: the scalar channels-last path
LAYOUTS = {"nchw": (24, False, 40), "nchw_t": (32, False, 3000), "cl8": (8, True, 3000),
           "cl64": (64, True, 3000), "cl160": (160, True, 3000), "cl12": (12, True, 3000)}


def _mapping(gen, B, H, W, Vw, msz, oob):
    counts = torch.randint(0, 4, (Vw,), generator=gen)
    counts[torch.rand(Vw, generator=gen) < 0.3] = 1
    aptr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)])
    P = int(aptr[-1])
    mw, mh = msz
    pix = torch.stack([torch.randint(0, mw, (P,), generator=gen), torch.randint(0, mh, (P,), generator=gen)], 1)
    pix[1::4] = pix[0:-1:4][: pix[1::4].shape[0]]                     # duplicated pixels
    pix[::7, 0] = mw - 1                                               # border
    if oob:
        pix[::29, 0] = mw + 5                                          # clamped like the forward
        pix[::31, 1] = -3
    img = torch.randint(0, B, (Vw,), generator=gen)
    return img, pix, aptr


def _run(fmap_nchw, dtype, cl, img, pix, aptr, reduce, msz, go):
    from deepviewagg_b200 import ops
    x = fmap_nchw.to(dtype)
    x = (x.permute(0, 2, 3, 1).contiguous() if cl else x).cuda().requires_grad_(True)
    if msz is None:
        out = ops.gather_pool(x, img.cuda(), pix.cuda(), aptr.cuda(), reduce, channels_last=cl)
    else:
        out = ops.interp_pool(x, img.cuda(), pix.cuda(), aptr.cuda(), msz, reduce=reduce, channels_last=cl)
    (gx,) = torch.autograd.grad(out, x, go.to(dtype).cuda())
    return (gx if cl else gx.permute(0, 2, 3, 1)).cpu()              # [B, H, W, C]


def _oracle(fmap_nchw, dtype, img, pix, aptr, reduce, msz, go):
    x = fmap_nchw.to(dtype).float().numpy()
    B, C, H, W = x.shape
    arg = None
    if reduce in ("max", "min"):
        arg = D.first_arg(D.gathered_values(x, img.numpy(), pix.numpy(), aptr.numpy(), msz), aptr.numpy(), reduce)
    g = go.to(dtype).float().numpy()
    ref = D.map_grad_ordered((B, H, W, C), g, img.numpy(), pix.numpy(), aptr.numpy(), reduce, arg, msz)
    return torch.from_numpy(ref).to(dtype)


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("interp", [False, True])
def test_map_grad_bit_exact_and_close_to_atomic(layout, interp):
    C, cl, Vw = LAYOUTS[layout]
    gen = torch.Generator().manual_seed(C + 7 * interp + Vw)
    B, H, W = 3, 19, 23
    msz = (2 * W + 3, 2 * H + 1) if interp else None
    img, pix, aptr = _mapping(gen, B, H, W, Vw, msz or (W, H), oob=not interp)
    fmap = torch.randn(B, C, H, W, generator=gen).relu()
    go = torch.randn(Vw, C, generator=gen)
    for reduce in ("sum", "mean", "max", "min"):
        for pdt in (torch.int16, torch.int32):
            for dt in (torch.float32, torch.bfloat16):
                what = f"{layout} interp={interp} {reduce} {pdt} {dt}"
                with deterministic():
                    got = _run(fmap, dt, cl, img, pix.to(pdt), aptr, reduce, msz, go)
                want = _oracle(fmap, dt, img, pix, aptr, reduce, msz, go)
                assert torch.equal(got, want), what
                atomic = _run(fmap, dt, cl, img, pix.to(pdt), aptr, reduce, msz, go)
                tol = 1e-6 if dt == torch.float32 else 8e-3
                assert rel_err(atomic.float(), got.float()) <= tol, what


@pytest.mark.parametrize("cl", [False, True])
def test_reuse_heavy_interp_bit_exact(cl):
    """Mapping at 4x the map resolution: hundreds of contributions per map pixel (buckets larger than
    a warp)."""
    gen = torch.Generator().manual_seed(11)
    B, C, H, W, P = 2, 64, 12, 10, 40000
    msz = (4 * W, 4 * H)
    img, pix, aptr = _mapping(gen, B, H, W, P // 2, msz, oob=False)
    fmap = torch.randn(B, C, H, W, generator=gen)
    go = torch.randn(aptr.numel() - 1, C, generator=gen)
    for reduce in ("sum", "max"):
        with deterministic():
            got = _run(fmap, torch.float32, cl, img, pix.int(), aptr, reduce, msz, go)
        assert torch.equal(got, _oracle(fmap, torch.float32, img, pix, aptr, reduce, msz, go)), reduce
        atomic = _run(fmap, torch.float32, cl, img, pix.int(), aptr, reduce, msz, go)
        # hundreds of signed terms per element: the two summation orders differ by more than 1e-6 of the
        # largest result, so bound the difference by the scale of the terms (sum of their magnitudes)
        scale = _oracle(fmap, torch.float32, img, pix, aptr, reduce, msz, go.abs())
        assert bool(((atomic - got).abs() <= 1e-6 * scale).all()), reduce


@pytest.mark.parametrize("cl", [False, True])
def test_sparse_interpolation_pixels_bit_exact(cl):
    from deepviewagg_b200 import ops
    g = load_golden("sparse_interpolation")
    W, H, _ = [int(v) for v in g["half_size"]]
    x = g["half_x"]
    B, C, h, w = x.shape
    pix, batch = g["half_pix"], g["half_batch"]
    go = torch.randn(pix.shape[0], C, generator=torch.Generator().manual_seed(2))
    xc = (x.permute(0, 2, 3, 1).contiguous() if cl else x).cuda().requires_grad_(True)
    with deterministic():
        out = ops.sparse_interpolation_pixels(xc, batch.cuda(), pix.int().cuda(), (W, H), channels_last=cl)
        (gx,) = torch.autograd.grad(out, xc, go.cuda())
    gx = (gx if cl else gx.permute(0, 2, 3, 1)).cpu()
    aptr = np.arange(pix.shape[0] + 1)
    want = D.map_grad_ordered((B, h, w, C), go.numpy(), batch.numpy(), pix.numpy(), aptr, "sum", None, (W, H))
    assert torch.equal(gx, torch.from_numpy(want))


def test_rows_scatter_add_bit_exact():
    """view_attention with a repeating row index: its x gradient is the rows scatter-add of the
    per-view gradient rows (those of the same call without index), in ascending view order."""
    from deepviewagg_b200 import ops
    gen = torch.Generator().manual_seed(4)
    N, C, G, R = 700, 64, 4, 300
    counts = torch.randint(0, 6, (N,), generator=gen)
    csr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)]).cuda()
    V = int(csr[-1])
    idx = torch.randint(0, R, (V,), generator=gen).cuda()             # every row feeds several views
    x = torch.randn(R, C, generator=gen).cuda()
    compat = torch.randn(V, G, generator=gen).cuda()
    go = torch.randn(N, C, generator=gen).cuda()
    xr = x[idx].clone().requires_grad_(True)
    out_rows = ops.view_attention(xr, compat, csr, G)[0]
    (g_rows,) = torch.autograd.grad(out_rows, xr, go)
    want = torch.from_numpy(D.scatter_add_rows_ordered(g_rows.cpu().numpy(), idx.cpu().numpy(), R))
    res = []
    for det in (True, True, False):
        xg = x.clone().requires_grad_(True)
        with deterministic(det):
            out = ops.view_attention(xg, compat, csr, G, idx=idx)[0]
            (gx,) = torch.autograd.grad(out, xg, go)
        res.append(gx.cpu())
    assert torch.equal(res[0], want) and torch.equal(res[1], want)
    assert rel_err(res[2], want) <= 1e-6
    # the helper directly: indices outside [0, R) skipped, bf16 rows, widths that are not 16-byte chunks
    for dt, Cw in ((torch.float32, 64), (torch.bfloat16, 64), (torch.float32, 13)):
        src = torch.randn(V, Cw, generator=gen).to(dt).cuda()
        ix = idx.clone()
        ix[::17] = R
        ix[::19] = -1
        with deterministic():
            got = ops._scatter_add_rows(src, ix, R).cpu()
        want = D.scatter_add_rows_ordered(src.float().cpu().numpy(), ix.cpu().numpy(), R)
        assert torch.equal(got, torch.from_numpy(want)), (dt, Cw)


def test_heuristic_pool_backward_under_flag():
    from deepviewagg_b200 import ops
    gen = torch.Generator().manual_seed(6)
    N, C = 500, 32
    counts = torch.randint(0, 5, (N,), generator=gen)
    csr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)]).cuda()
    V = int(csr[-1])
    x_mod = torch.randn(V, C, generator=gen).cuda()
    x_map = torch.randn(V, 3, generator=gen).cuda()
    go = torch.randn(N, C, generator=gen).cuda()
    res = []
    for det in (True, False):
        xm = x_mod.clone().requires_grad_(True)
        with deterministic(det):
            (g,) = torch.autograd.grad(ops.heuristic_pool(xm, x_map, csr, 1), xm, go)
        res.append(g)
    assert torch.equal(res[0], res[1])          # each point picks a distinct view: nothing is summed


def _branch_step(interpolate, channels_last):
    from test_containers import _toy_image_data
    from deepviewagg_b200.modules.multimodal.fusion import BimodalFusion
    from deepviewagg_b200.modules.multimodal.modules import UnimodalBranch
    from deepviewagg_b200.modules.multimodal.pooling import BimodalCSRPool, GroupBimodalCSRPool
    g = load_golden("unimodal_branch_interp" if interpolate else "unimodal_branch_toy")
    mod = _toy_image_data(g, "cuda")
    xs = []
    for im in mod:
        x = im.x.detach().clone()
        if channels_last:
            x = x.contiguous(memory_format=torch.channels_last)
        x.requires_grad_(True)
        im._x = x
        xs.append(x)
    view_pool = GroupBimodalCSRPool(in_map=8, in_mod=16, num_groups=4, use_num=True)
    view_pool.load_state_dict(g["sd"], strict=True)
    branch = UnimodalBranch(None, BimodalCSRPool(mode="max"), view_pool, BimodalFusion("concatenation"),
                            interpolate=interpolate).cuda()
    branch.train()
    x_3d = g["x_3d"].cuda().requires_grad_(True)
    out = branch({"x_3d": x_3d, "x_seen": None, "modalities": {"image": mod}}, "image")
    params = dict(view_pool.named_parameters())
    grads = torch.autograd.grad((out["x_3d"] * g["w"].cuda()).sum(), [x_3d] + xs + list(params.values()),
                                allow_unused=True)
    names = ["x_3d", "s0_x", "s1_x"] + ["param/" + k for k in params]
    return g, dict(zip(names, grads))


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("interpolate", [False, True])
def test_branch_training_step_reproducible(interpolate, channels_last):
    with deterministic():
        g, a = _branch_step(interpolate, channels_last)
        _, b = _branch_step(interpolate, channels_last)
    for n, ga in a.items():
        ref = g["grad"][n]
        if ga is None:
            assert b[n] is None and float(ref.abs().max()) == 0, n
            continue
        assert torch.equal(ga, b[n]), n
        assert (ga.cpu() - ref).abs().max() <= 2e-4 * max(1.0, float(ref.abs().max())), n


@pytest.mark.parametrize("interp", [False, True])
def test_large_map_grad_reproducible(interp):
    """About 1 M pixels with heavy pixel reuse: two runs are bit-identical."""
    from deepviewagg_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(8)
    B, C, H, W, P = 4, 64, 64, 96, 1_000_000
    msz = (4 * W, 4 * H) if interp else (W, H)
    pix = torch.stack([torch.randint(0, msz[0], (P,), device="cuda", generator=gen),
                       torch.randint(0, msz[1], (P,), device="cuda", generator=gen)], 1).to(torch.int16)
    counts = torch.randint(1, 4, (P // 2,), device="cuda", generator=gen)
    aptr = torch.cat([torch.zeros(1, dtype=torch.long, device="cuda"), counts.cumsum(0)])
    aptr = aptr[aptr <= P]
    pix = pix[: int(aptr[-1])]
    Vw = aptr.numel() - 1
    img = torch.randint(0, B, (Vw,), device="cuda", generator=gen)
    fmap = torch.randn(B, H, W, C, device="cuda", generator=gen)
    go = torch.randn(Vw, C, device="cuda", generator=gen)
    res = []
    with deterministic():
        for _ in range(2):
            x = fmap.clone().requires_grad_(True)
            if interp:
                out = ops.interp_pool(x, img, pix, aptr, msz, reduce="mean", channels_last=True)
            else:
                out = ops.gather_pool(x, img, pix, aptr, "mean", channels_last=True)
            res.append(torch.autograd.grad(out, x, go)[0])
    assert torch.equal(res[0], res[1])
