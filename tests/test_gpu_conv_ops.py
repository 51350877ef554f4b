"""Every kernel of libdva_conv2d.so, libdva_unet.so and libdva_resnet.so, one operator at a time, against float64.

Each case of tests/test_conv_ops_table.py runs its operator (the single-launch helpers of ops.py, or one C entry)
under the kernel recorder of tests/test_gpu_kernel_matrix.py, asserts by name that its kernels ran, checks every
output element by element with the bounds of that file on the kernel's own fp32 operands, checks the GEMM outputs
normwise against TAU, and runs again to assert bitwise reproducibility.  A kernel counts as checked once a case that
ran it has passed; test_every_kernel_checked asserts that all 44 are.

Also: the weight-standardisation gradient of constant and all-zero filters (finite, torch's masked std backward),
and a ResNetDown stack and a UNet whose standardised convolutions hold a zeroed filter, against the float64 oracles
with the bounds of tests/test_gpu_image_encoder.py / tests/test_gpu_image_unet.py."""
import math

import pytest
import torch

import test_conv2d_matrix_table as C2
import test_resnet18_matrix_table as CR
import test_unet_matrix_table as CU
from deepviewagg_b200 import ops
from deepviewagg_b200._lib import launch
from deepviewagg_b200.modules.multimodal.modalities import image as I
from test_conv_ops_table import (ALL_KERNELS, CASES, CASE_IDS, DEC_TAPS, ENC_TAPS, RELU_WS_SCALE, TINY, U32,
                                 bn_apply_ref, bn_bwd_ref, conv_bias, conv_bounds, conv_operands, gn_apply_ref, gn_bwd_ref,
                                 gn_groups, maxpool_ref, prep_filters, resize_ref, rho, standardized_grad_ref,
                                 standardized_ref, stats_ref, tau_of)
from test_gpu_kernel_matrix import record
from test_kernel_matrix_table import violations

pytestmark = pytest.mark.gpu
SEEN = set()
CHECKED = set()
RHO = {}          # (case id, output) -> normwise error of a GEMM output
EPS = 1e-5


def canon(name):
    return C2.canonical(name) or CU.canonical(name) or CR.canonical(name)


def check(what, got, ref, bound):
    n, msg = violations(got.contiguous(), ref.contiguous(), bound.contiguous())
    assert n == 0, f"{what}: {msg}"


def cpu(d):
    return {k: v.detach().cpu() for k, v in d.items()}


# ------------------------------------------------------------------------------------------------
# one operator per case: fn() -> dict of outputs (and the operands they were computed from)
# ------------------------------------------------------------------------------------------------
def _conv_fn(c):
    x, w, dz = conv_operands(c)
    bias = conv_bias(c)
    gen = torch.Generator().manual_seed(2)
    add = torch.randn(x.shape, generator=gen)
    xg, wg, dzg, bg, ag = (t.cuda() for t in (x, w, dz, bias, add))
    lib, geo, Ci, Co = c["lib"], c["geo"], c["Ci"], c["Co"]
    if lib == "resnet":
        rm0 = 0.1 * torch.randn(Co, generator=gen)
        rv0 = 0.5 + torch.rand(Co, generator=gen)

    def fn():
        if lib == "conv2d":
            T = ENC_TAPS[geo]
            wf, wd = ops._conv_weights(wg, geo, True)
            z, mean, invstd = ops._conv_fwd(xg, wf, bg, Co, geo, c["G"], EPS)
            z0 = ops._conv_fwd(xg, wf, torch.zeros_like(bg), Co, geo, c["G"], EPS)[0]
            dwf, db = ops._wgrad(dzg, xg, geo)
            dx = ops._dgrad(dzg, xg.shape, wd, geo, add=ag)
            dx0 = ops._dgrad(dzg, xg.shape, wd, geo)
            ws = wf.view(Co, T, T, Ci).permute(0, 3, 1, 2)
            dw = dwf.view(Co, T, T, Ci).permute(0, 3, 1, 2)
            return cpu(dict(ws=ws, z=z, z0=z0, mean=mean, invstd=invstd, dw=dw, db=db, dx=dx, dx0=dx0))
        if lib == "unet":
            T = DEC_TAPS[geo]
            wf, wd = ops._convt_weights(wg, geo)
            z, mean, invstd = ops._convt_fwd(xg, wf, bg, Co, geo, c["G"], EPS)
            z0 = ops._convt_fwd(xg, wf, torch.zeros_like(bg), Co, geo, c["G"], EPS)[0]
            dwf, db = ops._convt_wgrad(dzg, xg, geo)
            dx = ops._convt_dgrad(dzg, xg.shape, wd, geo, add=ag)
            dx0 = ops._convt_dgrad(dzg, xg.shape, wd, geo)
            ws = wd.view(Ci, T, T, Co).permute(0, 3, 1, 2)
            if T == 2:
                wsf, dw = (t.view(T, T, Co, Ci).permute(3, 2, 0, 1) for t in (wf, dwf))
            else:
                wsf, dw = (t.view(Co, T, T, Ci).flip(1, 2).permute(3, 0, 1, 2) for t in (wf, dwf))
            return cpu(dict(ws=ws, wsf=wsf, z=z, z0=z0, mean=mean, invstd=invstd, dw=dw, db=db, dx=dx, dx0=dx0))
        T = geo[0]
        rm, rv = rm0.cuda(), rv0.cuda()
        wf, wd = ops._rn_weights(wg)
        z, mean, invstd = ops._rn_conv_bn(xg, wf, Co, geo, (rm, rv, c["training"], 0.1, EPS))
        dw = ops._rn_wgrad(dzg, xg, Co, geo)
        dx = ops._rn_dgrad(dzg, xg.shape, wd, geo, add=ag)
        dx0 = ops._rn_dgrad(dzg, xg.shape, wd, geo)
        return cpu(dict(wf=wf.view(Co, T, T, Ci).permute(0, 3, 1, 2), wd=wd.view(Ci, T, T, Co).permute(3, 0, 1, 2),
                        z=z, mean=mean, invstd=invstd, rm=rm, rv=rv, dw=dw, dx=dx, dx0=dx0))
    return fn, dict(x=x, w=w, dz=dz, bias=bias, add=add, rm0=rm0 if lib == "resnet" else None,
                    rv0=rv0 if lib == "resnet" else None)


def _check_conv(c, out, opd):
    lib = c["lib"]
    if lib == "resnet":
        assert torch.equal(out["wf"], opd["w"]) and torch.equal(out["wd"], opd["w"]), "weight layouts"
        ws = out["wf"]
    else:
        ws = out["ws"]
        ref, bnd = standardized_ref(opd["w"])
        check("standardised filter", ws, ref, bnd)
        if lib == "unet":
            assert torch.equal(out["wsf"], ws), "the forward's and the data gradient's filters differ"
    refs = conv_bounds(c, opd["x"], ws, opd["dz"], bias=None if lib == "resnet" else opd["bias"], add=opd["add"])
    for k, (r, b) in refs.items():
        check(k, out[k], r, b)
    # normwise errors of the products alone: the forward without its bias (a bias of 10^3 would round z by far more
    # than the product errs), the data gradient without an addend
    plain = conv_bounds(c, opd["x"], ws, opd["dz"])
    z0 = out["z"] if lib == "resnet" else out["z0"]
    check("z without bias", z0, *plain["z"])
    check("dx without add", out["dx0"], *plain["dx"])
    RHO[(c["id"], "z")] = rho(z0, plain["z"][0])
    RHO[(c["id"], "dx")] = rho(out["dx0"], plain["dx"][0])
    RHO[(c["id"], "dw")] = rho(out["dw"], refs["dw"][0])
    z = out["z"]
    B = c["B"]
    if lib == "resnet":
        v = z.reshape(-1, c["Co"]).t()
        mu, inv, var, dmu, dinv, dvar = stats_ref(v, EPS)
        if c["training"]:
            check("mean", out["mean"], mu, dmu)
            check("invstd", out["invstd"], inv, dinv)
            n = v.shape[1]
            m = float(torch.tensor(0.1, dtype=torch.float32))     # the momentum as the kernel receives it
            rm = (1 - m) * opd["rm0"].double() + m * mu
            rv = (1 - m) * opd["rv0"].double() + m * var * n / (n - 1)
            check("running_mean", out["rm"], rm, m * dmu + U32 * rm.abs() + TINY)
            check("running_var", out["rv"], rv, m * dvar * n / (n - 1) + U32 * rv.abs() + TINY)
        else:
            assert torch.equal(out["mean"], opd["rm0"]) and torch.equal(out["rm"], opd["rm0"])
            assert torch.equal(out["rv"], opd["rv0"])
            inv_e = 1.0 / torch.sqrt(opd["rv0"].double() + EPS)
            check("eval invstd", out["invstd"], inv_e, U32 * inv_e)
    else:
        mu, inv, _, dmu, dinv, _ = stats_ref(gn_groups(z.reshape(B, -1, c["Co"]), c["G"]), EPS)
        check("mean", out["mean"].reshape(-1), mu, dmu)
        check("invstd", out["invstd"].reshape(-1), inv, dinv)
    for k in ("z", "dx", "dw"):
        assert RHO[(c["id"], k)] <= tau_of(c, k), (k, RHO[(c["id"], k)], tau_of(c, k))


def _prep_fn(c):
    w, g = prep_filters(c)
    wg = w.cuda()
    T = (ENC_TAPS if c["lib"] == "conv2d" else DEC_TAPS)[c["geo"]]
    if c["lib"] == "conv2d":
        dwf = g.permute(0, 2, 3, 1).contiguous().cuda()
    elif T == 2:
        dwf = g.permute(2, 3, 1, 0).contiguous().cuda()
    else:
        dwf = g.flip(2, 3).permute(1, 2, 3, 0).contiguous().cuda()

    def fn():
        if c["lib"] == "conv2d":
            Co, Ci = w.shape[:2]
            wf, wd = ops._conv_weights(wg, c["geo"], True)
            dw = ops._weight_grad(wg, dwf.view(-1), c["geo"], True)
            wsf = wf.view(Co, T, T, Ci).permute(0, 3, 1, 2)
            wsd = (wd.view(T, T, Ci, Co).permute(3, 2, 0, 1) if T == 2 else wd.view(Ci, T, T, Co).permute(3, 0, 1, 2))
        else:
            Ci, Co = w.shape[:2]
            wf, wd = ops._convt_weights(wg, c["geo"])
            dw = ops._convt_weight_grad(wg, dwf.view(-1), c["geo"])
            wsd = wd.view(Ci, T, T, Co).permute(0, 3, 1, 2)
            wsf = (wf.view(T, T, Co, Ci).permute(3, 2, 0, 1) if T == 2
                   else wf.view(Co, T, T, Ci).flip(1, 2).permute(3, 0, 1, 2))
        return cpu(dict(wsf=wsf, wsd=wsd, dw=dw))
    return fn, dict(w=w, g=g)


def _check_prep(c, out, opd):
    ref, bnd = standardized_ref(opd["w"])
    check("forward filter", out["wsf"], ref, bnd)
    assert torch.equal(out["wsd"], out["wsf"]), "the data gradient's filter differs"
    assert torch.isfinite(out["dw"]).all(), "non-finite weight gradient"
    ref, bnd = standardized_grad_ref(opd["w"], opd["g"])
    check("weight gradient", out["dw"], ref, bnd)


def _gn_fn(c):
    gen = torch.Generator().manual_seed(5)
    B, P, C, G = c["B"], c["P"], c["C"], c["G"]
    z = torch.randn(B, P, C, generator=gen) * 3 + 1

    def stats(t):
        v = gn_groups(t, G).double()
        return v.mean(1).float().reshape(B, G), (1 / torch.sqrt(v.var(1, unbiased=False) + EPS)).float().reshape(B, G)
    mean, inv = stats(z)
    gamma, beta = 1 + 0.3 * torch.randn(C, generator=gen), 0.3 * torch.randn(C, generator=gen)
    dy = torch.randn(B, P, C, generator=gen)
    skip = torch.randn(B, P, C, generator=gen) if c["skip"] else None
    ds = None
    if c["ds"]:
        zs = torch.randn(B, P, C, generator=gen)
        ds = (zs, *stats(zs), 1 + 0.3 * torch.randn(C, generator=gen), 0.3 * torch.randn(C, generator=gen))
    gp = lambda t: None if t is None else t.cuda()  # noqa: E731
    scale = RELU_WS_SCALE if c["relu"] else 0.0
    zg = z.view(B, 1, P, C).cuda()
    gn = (G, gp(mean), gp(inv), gp(gamma), gp(beta))
    dsg = None if ds is None else (ds[0].view(B, 1, P, C).cuda(), G, *(t.cuda() for t in ds[1:]))

    def fn():
        y = ops._gn_apply(zg, gn, c["relu"], skip=None if skip is None else skip.view(B, 1, P, C).cuda(), ds=dsg)
        dz, dgamma, dbeta = ops._gn_bwd(dy.view(B, 1, P, C).cuda(), zg, gn, c["relu"])
        return cpu(dict(y=y.view(B, P, C), dz=dz.view(B, P, C), dgamma=dgamma, dbeta=dbeta))
    return fn, dict(z=z, mean=mean, inv=inv, gamma=gamma, beta=beta, dy=dy, skip=skip, ds=ds, scale=scale)


def _check_gn(c, out, o):
    y, by = gn_apply_ref(o["z"], o["mean"], o["inv"], o["gamma"], o["beta"], c["G"], o["scale"], skip=o["skip"],
                         ds=o["ds"])
    check("y", out["y"], y, by)
    ref = gn_bwd_ref(o["dy"], o["z"], o["mean"], o["inv"], o["gamma"], o["beta"], c["G"], o["scale"])
    for k, (r, b) in ref.items():
        check(k, out[k], r, b)


def _bn_fn(c):
    gen = torch.Generator().manual_seed(6)
    M, C = c["M"], c["C"]
    z = torch.randn(M, C, generator=gen) * 2 - 0.5
    v = z.double()
    mean, inv = v.mean(0).float(), (1 / torch.sqrt(v.var(0, unbiased=False) + EPS)).float()
    gamma, beta = 1 + 0.3 * torch.randn(C, generator=gen), 0.3 * torch.randn(C, generator=gen)
    dy = torch.randn(M, C, generator=gen)
    skip = torch.randn(M, C, generator=gen) if c["skip"] else None
    ds = None
    if c["ds"]:
        zs = torch.randn(M, C, generator=gen)
        ds = (zs, zs.double().mean(0).float(), (1 / torch.sqrt(zs.double().var(0, unbiased=False) + EPS)).float(),
              1 + 0.3 * torch.randn(C, generator=gen), 0.3 * torch.randn(C, generator=gen))
    g4 = lambda t: t.view(1, 1, M, C).cuda()  # noqa: E731

    def fn():
        y = ops._rn_apply(g4(z), mean.cuda(), inv.cuda(), gamma.cuda(), beta.cuda(),
                          skip=None if skip is None else g4(skip),
                          ds=None if ds is None else (g4(ds[0]), *(t.cuda() for t in ds[1:])))
        dz, g, dgamma, dbeta = ops._rn_bn_bwd(g4(dy), y, g4(z), mean.cuda(), inv.cuda(), gamma.cuda(), c["training"],
                                             want_g=True)
        return cpu(dict(y=y.view(M, C), dz=dz.view(M, C), g=g.view(M, C), dgamma=dgamma, dbeta=dbeta))
    return fn, dict(z=z, mean=mean, inv=inv, gamma=gamma, beta=beta, dy=dy, skip=skip, ds=ds)


def _check_bn(c, out, o):
    y, by = bn_apply_ref(o["z"], o["mean"], o["inv"], o["gamma"], o["beta"], skip=o["skip"], ds=o["ds"])
    check("y", out["y"], y, by)
    ref = bn_bwd_ref(o["dy"], out["y"], o["z"], o["mean"], o["inv"], o["gamma"], c["training"])
    for k, (r, b) in ref.items():
        check(k, out[k], r, b)


def _act_fn(c):
    gen = torch.Generator().manual_seed(7)
    z, dy = torch.randn(c["n"], generator=gen), torch.randn(c["n"], generator=gen)
    z[:3] = torch.tensor([0.0, -0.0, 1e-30])

    def fn():
        zg, y, dz = z.cuda(), torch.empty(c["n"], device="cuda"), torch.empty(c["n"], device="cuda")
        launch("dva_unet_act", zg.device, zg, c["n"], RELU_WS_SCALE, y)
        launch("dva_unet_act_bwd", zg.device, dy.cuda(), zg, c["n"], RELU_WS_SCALE, dz)
        return cpu(dict(y=y, dz=dz))
    return fn, dict(z=z, dy=dy)


def _check_act(c, out, o):
    y = o["z"].double().clamp(min=0) * RELU_WS_SCALE
    dz = torch.where(o["z"] > 0, o["dy"].double() * RELU_WS_SCALE, torch.zeros(c["n"], dtype=torch.float64))
    # the scale is rounded to fp32, then one product: 2 u32
    check("y", out["y"], y, 2 * U32 * y.abs() + TINY)
    check("dz", out["dz"], dz, 2 * U32 * dz.abs() + TINY)


def _pool_fn(c):
    gen = torch.Generator().manual_seed(8)
    B, H, W, C = c["B"], c["H"], c["W"], c["C"]
    x = torch.randn(B, H, W, C, generator=gen)
    Ho, Wo = ops.rn_out(H, 2), ops.rn_out(W, 2)
    dy = torch.randn(B, Ho, Wo, C, generator=gen)

    def fn():
        xg = x.cuda()
        y = torch.empty(B, Ho, Wo, C, device="cuda")
        arg = torch.empty(B, Ho, Wo, C, dtype=torch.uint8, device="cuda")
        dx = torch.empty_like(xg)
        launch("dva_resnet_maxpool", xg.device, xg, B, H, W, C, y, arg)
        launch("dva_resnet_maxpool_bwd", xg.device, dy.cuda(), arg, B, H, W, C, dx)
        return cpu(dict(y=y, dx=dx))
    return fn, dict(x=x, dy=dy)


def _check_pool(c, out, o):
    y, grad = maxpool_ref(o["x"])
    assert torch.equal(out["y"].double(), y)
    dx = grad(o["dy"])
    check("dx", out["dx"], dx, 4 * U32 * grad(o["dy"].abs()) + TINY)


def _resize_fn(c):
    gen = torch.Generator().manual_seed(9)
    B, H, W, C, Ho, Wo = c["B"], c["H"], c["W"], c["C"], c["Ho"], c["Wo"]
    x = torch.randn(B, H, W, C, generator=gen)
    ld, col = C + 3, 2
    dy = torch.randn(B, Ho, Wo, ld, generator=gen)
    sh, sw = ops.resize_scale(H, Ho), ops.resize_scale(W, Wo)

    def fn():
        xg = x.cuda()
        y = torch.zeros(B, Ho, Wo, ld, device="cuda")
        dx = torch.empty_like(xg)
        launch("dva_resnet_resize", xg.device, xg, B, H, W, C, Ho, Wo, sh, sw, y, ld, col)
        launch("dva_resnet_resize_bwd", xg.device, dy.cuda(), ld, col, B, H, W, C, Ho, Wo, sh, sw, dx)
        return cpu(dict(y=y, dx=dx))
    return fn, dict(x=x, dy=dy[..., col:col + C].contiguous(), col=col)


def _check_resize(c, out, o):
    y, by, grad = resize_ref(o["x"], c["Ho"], c["Wo"])
    col, C = o["col"], c["C"]
    check("y", out["y"][..., col:col + C], y, by)
    assert not out["y"][..., :col].any() and not out["y"][..., col + C:].any(), "wrote outside its column slice"
    dx, bdx = grad(o["dy"])
    check("dx", out["dx"], dx, bdx)


RUN = {"conv": (_conv_fn, _check_conv), "prep": (_prep_fn, _check_prep), "gn": (_gn_fn, _check_gn),
       "bn": (_bn_fn, _check_bn), "act": (_act_fn, _check_act), "pool": (_pool_fn, _check_pool),
       "resize": (_resize_fn, _check_resize)}


def run_case(c):
    """Run one case under the recorder, check it, and run it again for bitwise reproducibility."""
    make, chk = RUN[c["op"]]
    fn, operands = make(c)
    out, names = record(fn, c["kernels"], canon=canon, seen=SEEN)
    for k in c["kernels"]:
        assert k in names, f"{k} did not run; recorded: {sorted(names)}"
    chk(c, out, operands)
    again = fn()
    for k, v in out.items():
        assert torch.equal(v, again[k]), f"{k} differs between two runs"
    CHECKED.update(c["kernels"])


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_case(case):
    run_case(case)


def test_every_kernel_checked():
    for c in CASES:
        if not set(c["kernels"]) <= CHECKED:
            run_case(c)
    assert CHECKED == ALL_KERNELS, {"never checked": sorted(ALL_KERNELS - CHECKED)}
    assert SEEN <= ALL_KERNELS, sorted(SEEN - ALL_KERNELS)


# ------------------------------------------------------------------------------------------------
# a zeroed filter through the modules
# ------------------------------------------------------------------------------------------------
def _zero_filters(net, cls):
    """Zero filter 0 and make filter 1 constant in every `cls` convolution of net."""
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, cls) and m.weight.shape[0] >= 2:
                m.weight[0] = 0.0
                m.weight[1] = 0.25


def test_resnet_down_with_a_zeroed_filter():
    from test_gpu_image_encoder import bounds, encoder, l2rel, maxrel, oracle_grads, run
    stages = encoder(4, seed=4)
    _zero_filters(stages, I.Conv2dWS)
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 48, 64, generator=gen).cuda()
    gy = torch.randn(2, 32, 3, 4, generator=gen).cuda()
    y, gx, gp = run(stages, x, gy)
    assert torch.isfinite(y).all() and torch.isfinite(gx).all() and all(torch.isfinite(g).all() for g in gp)
    ry, rgx, rgp = oracle_grads(stages, x, gy)
    by, bg = bounds(4)
    assert maxrel(y, ry) <= by
    assert l2rel(gx, rgx) <= bg
    for g, r in zip(gp, rgp):
        assert l2rel(g, r) <= bg


def test_unet_with_a_zeroed_filter():
    from test_gpu_image_unet import bounds, oracle_grads, perturbed, run
    from test_gpu_image_encoder import l2rel, maxrel
    from test_image_unet_oracle import small_opt
    torch.manual_seed(2)
    net = perturbed(I.UNet(small_opt("unet4", 4)), 3)
    up = next(m for m in net.modules() if isinstance(m, I.ConvTranspose2dWS))
    with torch.no_grad():
        up.weight[0] = 0.0                  # the filter of input channel 0 of the first ResNetUp
    net = net.cuda()
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 48, 64, generator=gen).cuda()
    gy = torch.randn(2, 13, 48, 64, generator=gen).cuda()
    y, gx, gp = run(net, x, gy)
    assert torch.isfinite(y).all() and torch.isfinite(gx).all() and all(torch.isfinite(g).all() for g in gp)
    ry, rgx, rgp = oracle_grads(net, x, gy, "unet4")
    by, bg = bounds(4)
    assert maxrel(y, ry) <= by
    assert l2rel(gx, rgx) <= bg
    for g, r in zip(gp, rgp):
        assert l2rel(g, r) <= bg
