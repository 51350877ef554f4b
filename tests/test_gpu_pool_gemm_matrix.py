"""Every feature-map pool, BatchNorm + LeakyReLU and projection GEMM instantiation, launched and proven launched:
each configuration runs under torch.profiler and asserts, by demangled kernel name, every table kernel it must
launch; results are checked element by element against float64 with the bounds of
tests/test_pool_gemm_matrix_table.py."""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from test_gpu_kernel_matrix import place, record as _record
from test_kernel_matrix_table import DTYPES, V16, kname, round_to, violations
from test_pool_gemm_matrix_table import (CASE_IDS, CASES, LAYER, POOL_CONFS, SK, bn_configs, bn_inputs,
                                         bn_launches, bn_reference, canonical, dw_chain, gemm_bound, pool_backward_ref,
                                         pool_det_ref, pool_forward_ref, pool_inputs, pool_launches)

pytestmark = pytest.mark.gpu
SEEN = set()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def record(fn, want=()):
    return _record(fn, want, canon=canonical, seen=SEEN)


def _reset_to(*tensors):
    """A function that puts `tensors` back to their values of now.  The recorder runs a session body again when a
    kernel record is missing, so a body that updates running buffers in place calls it first: every run then starts
    from the same state and takes exactly one momentum step."""
    saved = [t.detach().clone() for t in tensors]

    def reset():
        with torch.no_grad():
            for t, s in zip(tensors, saved):
                t.copy_(s)
    return reset


def assert_ran(kernels, names):
    missing = sorted(set(kernels) - names)
    assert not missing, f"{missing} did not run; recorded: {sorted(names)}"


def check(what, got, ref, bound, bad=None):
    n, msg = violations(got, ref, bound)
    if bad is not None:
        if n:
            bad[what] = msg
        return
    assert n == 0, f"{what}: {msg}"


# ------------------------------------------------------------------------------------------------
# feature-map pools
# ------------------------------------------------------------------------------------------------
def run_pool(conf):
    from deepviewagg_b200 import ops
    inp = pool_inputs(conf)
    ref, bnd, arg = pool_forward_ref(inp)
    gref, gbnd = pool_backward_ref(inp, arg)
    gdet = pool_det_ref(inp, arg)
    fmap = inp["x"].permute(0, 2, 3, 1).contiguous() if inp["cl"] else inp["x"]
    fm = place(fmap, inp["off"]).requires_grad_(True)
    img, pix, ptr = inp["images"].cuda(), inp["pixels"].cuda(), inp["ptr"].cuda()
    gout = inp["gout"].cuda()

    def go():
        if inp["interp"]:
            out = ops.interp_pool(fm, img, pix, ptr, inp["msz"], reduce=inp["red"], channels_last=inp["cl"])
        else:
            out = ops.gather_pool(fm, img, pix, ptr, reduce=inp["red"], channels_last=inp["cl"])
        ga, = torch.autograd.grad(out, fm, gout, retain_graph=True)
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)
        try:
            gd, = torch.autograd.grad(out, fm, gout)
        finally:
            torch.use_deterministic_algorithms(prev)
        return out, ga, gd
    want = pool_launches(conf)
    (out, ga, gd), names = record(go, want)
    assert_ran(want, names)
    if conf[2] == "nchw_t":
        assert not any(n.startswith("gather_pool_fwd_kernel") for n in names), sorted(names)
    out = out.cpu().double()
    if bnd is None:
        assert torch.equal(out, ref), f"{inp['red']}: {violations(out, ref, torch.zeros_like(ref))[1]}"
    else:
        check(inp["red"], out, ref, bnd)
    one = inp["counts"] == 1
    vals_one = ref[one] if bnd is None else round_to(ref[one], inp["dtype"])
    assert torch.equal(out[one], vals_one), "one-pixel views are copies"
    assert (out[inp["counts"] == 0] == 0).all(), "empty views are zeros"
    to_bhwc = (lambda t: t) if inp["cl"] else (lambda t: t.permute(0, 2, 3, 1))
    assert ga.dtype == fm.dtype and gd.dtype == fm.dtype
    check("atomic map gradient", to_bhwc(ga.cpu()), gref, gbnd)
    got = to_bhwc(gd.cpu()).double()
    if not torch.equal(got, gdet):
        pytest.fail(f"deterministic map gradient: {violations(got, gdet, torch.zeros_like(gdet))[1]}")


POOL_IDS = [f"{dt}-{pix}-{route}-{('sum', 'mean', 'max', 'min')[red]}-{'interp' if i else 'gather'}"
            for dt, pix, route, red, i in POOL_CONFS]


@pytest.mark.parametrize("conf", POOL_CONFS, ids=POOL_IDS)
def test_pool_configuration(conf):
    run_pool(conf)


# ------------------------------------------------------------------------------------------------
# BatchNorm + LeakyReLU
# ------------------------------------------------------------------------------------------------
def run_bn(dt, vec, cfg):
    from deepviewagg_b200 import ops
    inp = bn_inputs(dt, cfg)
    R, C = cfg["R"], cfg["C"]
    bn = torch.nn.BatchNorm1d(C, momentum=cfg["momentum"], affine=cfg["affine"]).cuda()
    with torch.no_grad():
        if cfg["affine"]:
            bn.weight.copy_(inp["gamma"]), bn.bias.copy_(inp["beta"])
        bn.running_mean.copy_(inp["rm"]), bn.running_var.copy_(inp["rv"])
        bn.num_batches_tracked.fill_(inp["tracked"])
    bn.train(cfg["training"])
    z = place(inp["z"], cfg["z_off"]).requires_grad_(True)
    dy = inp["dy"].cuda()
    leaves = [z] + ([bn.weight, bn.bias] if cfg["affine"] else [])
    reset = _reset_to(bn.running_mean, bn.running_var, bn.num_batches_tracked)

    def go():
        reset()
        y = ops.batch_norm_act(z, bn, negative_slope=0.2)
        return (y,) + torch.autograd.grad(y, leaves, dy)
    want = bn_launches(dt, vec, cfg["training"])
    res, names = record(go, want)
    assert_ran(want, names)
    ref = bn_reference(inp, vec)
    what = f"{dt} vec={vec} {cfg}"
    check(f"y {what}", res[0], ref["y"], ref["b_y"])
    check(f"dz {what}", res[1], ref["dz"], ref["b_dz"])
    if cfg["affine"]:
        check(f"d gamma {what}", res[2], ref["dgamma"], ref["b_dgamma"])
        check(f"d beta {what}", res[3], ref["dbeta"], ref["b_dbeta"])
    if cfg["training"]:
        check(f"running mean {what}", bn.running_mean, ref["rm"], ref["b_rm"])
        check(f"running var {what}", bn.running_var, ref["rv"], ref["b_rv"])
    else:
        assert torch.equal(bn.running_mean.cpu(), inp["rm"]), "eval leaves the running buffers alone"
    return names


BN_PARAMS = [(dt, vec) for dt in DTYPES for vec in (V16[dt], 1)]


@pytest.mark.parametrize("dt,vec", BN_PARAMS, ids=[f"{d}-vec{v}" for d, v in BN_PARAMS])
def test_bn_configuration(dt, vec):
    for cfg in bn_configs(dt, vec):
        run_bn(dt, vec, cfg)


# ------------------------------------------------------------------------------------------------
# projection GEMMs
# ------------------------------------------------------------------------------------------------
def _dw_family(names):
    if "tc::tc_dw_kernel" in names:
        return "tc"
    if "skinny_dw_kernel" in names:
        return "ffma"
    return "mma"


def run_linear(shape, seed=0, bad=None, want=()):
    """ops.linear forward + backward of one (M, K, N, x offset) under the recorder; bounds checked (violations
    collected into `bad` when given, else asserted)."""
    from deepviewagg_b200 import ops
    M, K, N, off = shape
    gen = torch.Generator().manual_seed(seed + M + 7 * K + 13 * N)
    x0 = torch.randn(M, K, generator=gen)
    w0 = torch.randn(N, K, generator=gen) / math.sqrt(K)
    g0 = torch.randn(M, N, generator=gen)
    x = place(x0, off).requires_grad_(True)
    w = w0.cuda().requires_grad_(True)
    g = g0.cuda()

    def go():
        y = ops.linear(x, w)
        return (y,) + torch.autograd.grad(y, [x, w], g)
    (y, gx, gw), names = record(go, want)
    x64, w64, g64 = x0.double(), w0.double(), g0.double()
    Kp, Np = K + (-K) % 4, N + (-N) % 4                 # ops.linear zero-pads wide layers: longer chains
    tag = f"{shape}"
    check(f"linear {tag}", y, x64 @ w64.t(), gemm_bound(x64.abs() @ w64.abs().t(), Kp), bad)
    check(f"linear dX {tag}", gx, g64 @ w64, gemm_bound(g64.abs() @ w64.abs(), Np), bad)
    L = dw_chain(_dw_family(names), M, Np, Kp)
    check(f"linear dW {tag}", gw, g64.t() @ x64, gemm_bound(g64.abs().t() @ x64.abs(), L), bad)
    return names


def run_layer(shape, seed=0, want=()):
    """ops.linear_bn_act (training, LeakyReLU 0.2) forward + backward against the float64 chain: the GEMM bound of
    z feeds the BatchNorm bounds; dX and dW add the propagated error of dz."""
    from deepviewagg_b200 import ops
    M, K, N, off = shape
    gen = torch.Generator().manual_seed(seed + M + 7 * K + 13 * N)
    x0 = torch.randn(M, K, generator=gen) * 1.5 + 0.3
    x0[:, 0] = 40.0 + 0.05 * torch.randn(M, generator=gen)       # columns of z with |mean| / std up to ~1e2 - 1e3
    w0 = torch.randn(N, K, generator=gen) / math.sqrt(K)
    w0[: N // 2, 0] = 5.0
    bn = torch.nn.BatchNorm1d(N, momentum=0.1).cuda()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(N, generator=gen) + 0.5)
        bn.bias.copy_(torch.randn(N, generator=gen) * 0.3)
        bn.running_mean.copy_(torch.randn(N, generator=gen)), bn.running_var.copy_(torch.rand(N, generator=gen) + 0.5)
    gamma, beta, rm0, rv0 = (bn.weight.detach().cpu().clone(), bn.bias.detach().cpu().clone(),
                             bn.running_mean.cpu().clone(), bn.running_var.cpu().clone())
    dy0 = torch.randn(M, N, generator=gen)
    x = place(x0, off).requires_grad_(True)
    w = w0.cuda().requires_grad_(True)
    reset = _reset_to(bn.running_mean, bn.running_var, bn.num_batches_tracked)

    def go():
        reset()
        y = ops.linear_bn_act(x, w, bn, negative_slope=0.2)
        return (y,) + torch.autograd.grad(y, [x, w, bn.weight, bn.bias], dy0.cuda())
    (y, gx, gw, gg, gb), names = record(go, want)
    x64, w64 = x0.double(), w0.double()
    z = x64 @ w64.t()
    dzin = gemm_bound(x64.abs() @ w64.abs().t(), K)
    inp = dict(z=z, gamma=gamma, beta=beta, rm=rm0, rv=rv0, dy=dy0, eps=bn.eps, momentum=0.1, tracked=0,
               training=True, dtype="f32")
    ref = bn_reference(inp, 4, dzin=dzin, epilogue=True)
    tag = f"layer {shape}"
    check(f"{tag} y", y, ref["y"], ref["b_y"])
    check(f"{tag} d gamma", gg, ref["dgamma"], ref["b_dgamma"])
    check(f"{tag} d beta", gb, ref["dbeta"], ref["b_dbeta"])
    check(f"{tag} running mean", bn.running_mean, ref["rm"], ref["b_rm"])
    check(f"{tag} running var", bn.running_var, ref["rv"], ref["b_rv"])
    dz, bdz = ref["dz"], ref["b_dz"]
    check(f"{tag} dX", gx, dz @ w64, gemm_bound(dz.abs() @ w64.abs(), N, bdz @ w64.abs()))
    fam = "mlp" if any(n.startswith("mlp_layer_bwd_kernel") for n in names) else _dw_family(names)
    check(f"{tag} dW", gw, dz.t() @ x64, gemm_bound(dz.abs().t() @ x64.abs(), dw_chain(fam, M, N, K),
                                                    bdz.t() @ x64.abs()))
    return names


def run_bnstats(shape):
    """dva_linear_bnstats_fwd directly: mean, invstd and the running buffers of z = x w^T from the GEMM epilogue."""
    from deepviewagg_b200 import ops
    M, K, N, off = shape
    gen = torch.Generator().manual_seed(M + K + N)
    x0 = torch.randn(M, K, generator=gen)
    x0[:, 0] = 100.0 + 0.02 * torch.randn(M, generator=gen)
    w0 = torch.randn(N, K, generator=gen) / math.sqrt(K)
    w0[::3, 0] = 10.0                                  # mean ~ 1e3, std ~ 1: the per-CTA shifts matter
    rm, rv = torch.randn(N, generator=gen).cuda(), (torch.rand(N, generator=gen) + 0.5).cuda()
    rm0, rv0 = rm.cpu().clone(), rv.cpu().clone()
    reset = _reset_to(rm, rv)

    def go():
        reset()
        return ops._linear_bnstats(place(x0, off), w0.cuda(), rm, rv, 0.1, 1e-5)
    (z, mean, invstd), names = record(go, ("tc::bn_stats_finalize_kernel",))
    x64, w64 = x0.double(), w0.double()
    inp = dict(z=x64 @ w64.t(), gamma=None, beta=None, rm=rm0, rv=rv0, dy=torch.zeros(M, N), eps=1e-5,
               momentum=0.1, tracked=0, training=True, dtype="f32")
    ref = bn_reference(inp, 4, dzin=gemm_bound(x64.abs() @ w64.abs().t(), K), epilogue=True)
    check(f"bnstats z {shape}", z, inp["z"], gemm_bound(x64.abs() @ w64.abs().t(), K))
    check(f"bnstats mean {shape}", mean, ref["mu"], ref["dmu"] + 2.0 ** -126)
    check(f"bnstats invstd {shape}", invstd, ref["inv"], ref["dinv"] + 2.0 ** -126)
    check(f"bnstats running mean {shape}", rm, ref["rm"], ref["b_rm"])
    check(f"bnstats running var {shape}", rv, ref["rv"], ref["b_rv"])
    return names


def ffma_child():
    """Body of the DVA_SKINNY=ffma child process: the fp32-pipe skinny cases under the recorder."""
    bad, names = {}, set()
    want = (kname("skinny_rows_kernel", True), kname("skinny_rows_kernel", False), "skinny_dw_kernel",
            "skinny_dw_reduce_kernel")
    for key in ("A", "G", "D"):
        names |= run_linear(SK[key], bad=bad, want=want)
    return dict(names=sorted(names), bad=bad)


def run_ffma_child():
    code = ("import json, sys\n"
            f"sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
            "import test_gpu_pool_gemm_matrix as T\n"
            "print('FFMA_RESULT ' + json.dumps(T.ffma_child()))\n")
    env = dict(os.environ, DVA_SKINNY="ffma")
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("FFMA_RESULT ")][-1]
    res = json.loads(line[len("FFMA_RESULT "):])
    SEEN.update(res["names"])
    return set(res["names"]), res["bad"]


@pytest.fixture(scope="module")
def ffma_result():
    return run_ffma_child()


GEMM_CASES = [c for c in CASES if c["kind"] == "gemm"]


def run_gemm_case(case, ffma_result=None):
    from deepviewagg_b200 import ops
    if case["ffma"]:
        names, bad = ffma_result if ffma_result is not None else run_ffma_child()
        assert not bad, bad
        assert_ran({case["kernel"]}, names)
        return
    names, want = set(), (case["kernel"],)
    for shape in case["shapes"]:
        if case["via"] == "linear":
            names |= run_linear(shape, want=want)
        elif case["kernel"] == "tc::bn_stats_finalize_kernel":
            names |= run_bnstats(shape) | run_layer(shape, want=want)
        else:
            old = ops._MLP_LAYER_FUSED["max_k"]
            ops._MLP_LAYER_FUSED["max_k"] = 64 if shape == LAYER["L64"] else old
            try:
                names |= run_layer(shape, want=want)
            finally:
                ops._MLP_LAYER_FUSED["max_k"] = old
    assert_ran({case["kernel"]}, names)


@pytest.mark.parametrize("case", GEMM_CASES, ids=[c["kernel"] for c in GEMM_CASES])
def test_gemm_instantiation(case, request):
    run_gemm_case(case, request.getfixturevalue("ffma_result") if case["ffma"] else None)


@pytest.mark.parametrize("shape", [(3000, 128, 128, 1), (1000, 16, 8, 1), (2999, 64, 96, 3)])
def test_misaligned_input_linear(shape):
    """A contiguous fp32 input at an odd storage offset: the wgmma shapes copy it to an aligned buffer, the skinny
    kernels read it in place with scalar loads; forward and backward within the GEMM bounds."""
    M, K, N, _ = shape
    wide = K > 64 or N > 64
    names = run_linear(shape, want=("tc::tc_rows_kernel<true>", "tc::tc_dw_kernel") if wide else ())
    if wide:
        assert "tc::tc_rows_kernel<true>" in names and "tc::tc_dw_kernel" in names, names


@pytest.mark.parametrize("shape,fused", [((3000, 128, 128, 1), False), ((1000, 128, 96, 1), False),
                                         ((5000, 32, 32, 1), True), ((3001, 8, 32, 1), True)])
def test_misaligned_input_linear_bn_act(shape, fused):
    names = run_layer(shape, want=("tc::bn_stats_finalize_kernel",))
    assert any(n.startswith("mlp_layer_bwd_kernel") for n in names) == fused, sorted(names)
    assert "tc::bn_stats_finalize_kernel" in names


def test_stateful_session_bodies_are_repeatable(monkeypatch):
    """Every session body that updates running buffers gives the single-step results when the recorder runs it
    twice (as it does when a kernel record goes missing)."""
    once = record

    def twice(fn, want=()):
        fn()
        return once(fn, want)
    monkeypatch.setattr(sys.modules[__name__], "record", twice)
    run_bn("f32", 4, bn_configs("f32", 4)[0])
    run_bn("f32", 4, bn_configs("f32", 4)[2])          # momentum None: the cumulative average's factor must not move
    run_layer(LAYER["L32"])
    run_layer(LAYER["W"])
    run_bnstats(LAYER["W"])


def test_every_instantiation_launched(ffma_result):
    """The union of the kernels recorded by all configurations is exactly the case table (configurations not run
    yet in this session, e.g. under -k, are run here)."""
    table = set(CASE_IDS)
    for conf in POOL_CONFS:
        if not pool_launches(conf) <= SEEN:
            try:
                run_pool(conf)
            except AssertionError:
                pass
    for dt, vec in ((d, v) for d in DTYPES for v in (V16[d], 1)):
        if not bn_launches(dt, vec, True) <= SEEN:
            for cfg in bn_configs(dt, vec):
                try:
                    run_bn(dt, vec, cfg)
                except AssertionError:
                    pass
    for case in GEMM_CASES:
        if case["kernel"] not in SEEN:
            try:
                run_gemm_case(case, ffma_result)
            except AssertionError:
                pass
    assert SEEN == table, {"never launched": sorted(table - SEEN), "launched without a case": sorted(SEEN - table)}
