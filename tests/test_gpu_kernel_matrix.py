"""Every view-attention, segment and qk_scores instantiation, launched and proven launched: each case runs
under torch.profiler (CUDA activity tracing only) and asserts, by demangled kernel name, that its
instantiation ran; results are checked element by element against the float64 oracle with the bounds of
tests/test_kernel_matrix_table.py."""
import functools
import time

import pytest
import torch

from oracle.scatter_standin import segment_csr as S_segment_csr, segment_csr_arg as S_segment_csr_arg
from oracle import pooling_oracle as O
from test_kernel_matrix_table import (CASES, CASE_IDS, DTYPES, K_ERR, TINY, U32, U_S, V16, VA_VARIANTS,
                                      canonical, kname, ptr_of, segment_counts, va_bounds, va_inputs,
                                      va_reference, violations)

pytestmark = pytest.mark.gpu
SEEN = set()
RED_NAMES = ("sum", "mean", "max", "min")


RECORD_ATTEMPTS = 8


def _lead_in():
    """A few sacrificial launches and a short pause at the start of a profiler session, before the kernels under
    test."""
    t = torch.zeros(1, device="cuda")
    for _ in range(16):
        t.add_(1)
    torch.cuda.synchronize()
    time.sleep(0.05)


def record(fn, want=(), canon=canonical, seen=SEEN):
    """Run fn() under the profiler; returns (fn's result, set of canonical dva kernel names that ran).
    canon: demangled name -> canonical name of a listed family, or None; seen: the set every recorded name joins.

    The profiler is a lossy observer: under host CPU load, about 1 - 2 % of short sessions come back with
    some or all of their kernel records missing (measured on an H100 over 300-session runs; pausing before
    or after the session, or keeping CUPTI attached between sessions, does not change the rate), and losses
    can come several sessions in a row.  So fn() is run again, after a growing pause, while a name in `want`
    is missing, at most RECORD_ATTEMPTS times.  The dispatch is deterministic and a name is only recorded
    when its kernel ran, so the union over the runs never reports a kernel that did not run: a silent
    fallback is missing from every run and still fails.  fn() must therefore give the same result every time it
    runs (a body that updates state in place restores it first).

    Every session starts with a lead-in (_lead_in): late in a long test process the profiler was seen to drop
    the records of the kernels launched first in a session, in every retry, while keeping the later ones."""
    from torch.profiler import ProfilerActivity, profile
    names, active = set(), False
    for attempt in range(RECORD_ATTEMPTS):
        if attempt:
            time.sleep(0.05 * attempt)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _lead_in()
            res = fn()
            torch.cuda.synchronize()
        evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        active |= bool(evs)
        names |= {k for k in (canon(e.name) for e in evs) if k is not None}
        if all(w in names for w in want):
            break
    if not active:
        pytest.fail("the profiler recorded no CUDA activity: kernel names cannot be checked")
    seen.update(names)
    return res, names


def assert_ran(kernel, names):
    assert kernel in names, f"{kernel} did not run; recorded: {sorted(names)}"


def place(t, off):
    """t on the GPU at a storage offset of `off` elements (off = 1: not 16-byte aligned)."""
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device="cuda")
    buf[off:].copy_(t.reshape(-1))
    return buf[off:].view(t.shape)


def check(what, got, ref, bound):
    n, msg = violations(got, ref, bound)
    assert n == 0, f"{what}: {msg}"


@pytest.fixture
def va_path():
    from deepviewagg_b200 import _lib
    lib = _lib.load()

    def set_path(p):
        assert lib.dva_view_attention_set_path(p) == 0
    yield set_path
    set_path(0)


# ------------------------------------------------------------------------------------------------
# view attention
# ------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=3)
def va_expected(dtype, C, G, variant):
    """Inputs, float64 reference and bounds of one shape (shared by the ring, lane and streaming cases)."""
    inp = va_inputs(dict(dtype=dtype, C=C, G=G), variant)
    ref = va_reference(inp)
    return inp, ref, va_bounds(inp, ref)


def run_va(inp, x_off=0, c_off=0, want=()):
    """One forward + backward on the GPU under the recorder: ((results), kernel names)."""
    from deepviewagg_b200 import ops
    x = place(inp["x"], x_off).requires_grad_(True)
    c = place(inp["compat"], c_off).requires_grad_(True)
    gw = inp["gw"].cuda().requires_grad_(True) if inp["gw"] is not None else None
    gb = inp["gb"].cuda().requires_grad_(True) if inp["gb"] is not None else None
    gout = inp["gout"].cuda()

    def go():
        out, att, smax = ops.view_attention(x, c, inp["ptr"].cuda(), inp["G"],
                                            idx=None if inp["idx"] is None else inp["idx"].cuda(),
                                            gate_weight=gw, gate_bias=gb, group_scaling=inp["scaling"],
                                            idx_is_permutation=inp["is_perm"])
        leaves = [x, c] + ([gw, gb] if gw is not None else [])
        return (out, att, smax) + tuple(torch.autograd.grad(out, leaves, gout))
    return record(go, want)


def check_va(res, inp, ref=None, bnd=None):
    if ref is None:
        ref = va_reference(inp)
        bnd = va_bounds(inp, ref)
    out, att, smax, gx, gc = res[:5]
    check("out", out, ref["out"], bnd["out"])
    check("attentions", att, ref["att"], bnd["att"])
    ptr = inp["ptr"]
    empty = (ptr[1:] == ptr[:-1]).cuda()
    assert (out[empty] == 0).all(), "unseen points must be exact zeros"
    grp = torch.repeat_interleave(torch.arange(inp["G"]), torch.tensor(O.group_sizes(out.shape[1], inp["G"])))
    closed = bnd["closed"][:, grp].cuda()
    assert (out[closed] == 0).all(), "gated-out groups must be exact zeros"
    m_ref = S_segment_csr(inp["compat"], ptr, reduce="max")
    assert torch.equal(smax.cpu()[~empty.cpu()], m_ref[~empty.cpu()]), "segment max must be bit-exact"
    check("grad_x", gx, ref["gx"], bnd["gx"])
    check("grad_compat", gc, ref["gcompat"], bnd["gcompat"])
    if len(res) > 5:
        check("grad_gate_w", res[5], ref["gw"], bnd["gw"])
        check("grad_gate_b", res[6], ref["gb"], bnd["gb"])


VA_CASES = [c for c in CASES if c["kind"] == "va"]


def _run_case(case, va_path):
    kind = case["kind"]
    if kind == "va":
        va_path(case["path"])
        for variant in range(len(VA_VARIANTS)):
            inp, ref, bnd = va_expected(case["dtype"], case["C"], case["G"], variant)
            res, names = run_va(inp, case["x_off"], case["c_off"], want=(case["kernel"],))
            assert_ran(case["kernel"], names)
            check_va(res, inp, ref, bnd)
    else:
        RUNNERS[kind](case)


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_instantiation(case, va_path):
    _run_case(case, va_path)


def test_recorder_catches_a_silent_fallback(va_path):
    """A ring-eligible shape with the streaming path forced: the recorder sees streaming kernels, and the
    ring case's own assertion rejects that run."""
    case = next(c for c in VA_CASES if c["kernel"] == kname("va_ring_fwd_kernel", "float", 16))
    va_path(1)
    inp, ref, bnd = va_expected(case["dtype"], case["C"], case["G"], 0)
    streaming = (kname("view_attention_fwd_kernel", "float", 4, 16, 1, 4),
                 kname("view_attention_bwd_kernel", "float", 4, 16, 1, 4, True))
    res, names = run_va(inp, want=streaming)
    assert all(k in names for k in streaming), names
    assert not any(n.startswith("va_ring") or n.startswith("va_lane") for n in names), names
    with pytest.raises(AssertionError):
        assert_ran(case["kernel"], names)
    check_va(res, inp, ref, bnd)


@pytest.mark.parametrize("dt,C,long_segments,expect,reject", [
    # short segments (<= 12 views per point on average): ring forward; 128-byte rows: lane backward
    ("f32", 32, False, [kname("va_ring_fwd_kernel", "float", 8), kname("va_lane_bwd_kernel", "float", 8)],
     ["va_ring_bwd_kernel", "view_attention_"]),
    # 256-byte rows: ring backward
    ("f32", 64, False, [kname("va_ring_fwd_kernel", "float", 16), kname("va_ring_bwd_kernel", "float", 16)],
     ["va_lane_bwd_kernel", "view_attention_"]),
    # more than 12 views per point: streaming forward, lane backward
    ("bf16", 64, True, [kname("view_attention_fwd_kernel", "__nv_bfloat16", 8, 8, 1, 4),
                        kname("va_lane_bwd_kernel", "__nv_bfloat16", 8)], ["va_ring", "view_attention_bwd"]),
])
def test_auto_path_choice(dt, C, long_segments, expect, reject, va_path):
    va_path(0)
    inp = dict(va_inputs(dict(dtype=dt, C=C, G=4), 0))
    if long_segments:
        gen = torch.Generator().manual_seed(5)
        counts = 13 + torch.poisson(torch.full((400,), 8.0), generator=gen).long()
        ptr = ptr_of(counts)
        V = int(ptr[-1])
        inp.update(ptr=ptr, x=torch.randn(V, C, generator=gen).to(DTYPES[dt]),
                   compat=torch.randn(V, 4, generator=gen), gout=torch.randn(400, C, generator=gen).to(DTYPES[dt]))
    res, names = run_va(inp, want=expect)
    for k in expect:
        assert_ran(k, names)
    for prefix in reject:
        assert not any(n.startswith(prefix) for n in names), (prefix, sorted(names))
    check_va(res, inp)


# ------------------------------------------------------------------------------------------------
# segment primitives
# ------------------------------------------------------------------------------------------------
def _seg_confs(dt, vec):
    """(K, storage offset) of the inputs routed to `vec`: K a multiple of the vector width, aligned; or odd K;
    or a multiple of the vector width one element off 16-byte alignment."""
    return [(3 * V16[dt], 0)] if vec > 1 else [(7, 0), (2 * V16[dt], 1)]


def _seg_values(gen, dt, V, K):
    x = (torch.randn(V, K, generator=gen) * 3).to(DTYPES[dt])
    x[1::9] = x[0::9][:x[1::9].shape[0]]                     # ties: the first row must win
    return x


def _sum_bound(dt, absx, ptr, ref, mean=False):
    """u_s |ref| + K u32 (n + 1) sum |x| (over n for a mean)."""
    n = (ptr[1:] - ptr[:-1]).double().view(-1, 1)
    acc = K_ERR * U32 * (n + 1) * S_segment_csr(absx, ptr, reduce="sum")
    return U_S[dt] * ref.abs() + (acc / n.clamp(min=1) if mean else acc) + TINY[dt]


def run_segment_csr(case):
    from deepviewagg_b200 import ops
    dt, red = case["dtype"], RED_NAMES[case["red"]]
    gen = torch.Generator().manual_seed(11 + case["red"])
    ptr = ptr_of(segment_counts(gen, 300))
    V, ran = int(ptr[-1]), set()
    for K, off in _seg_confs(dt, case["vec"]):
        x = _seg_values(gen, dt, V, K)
        gout = torch.randn(ptr.numel() - 1, K, generator=gen).to(DTYPES[dt])
        xg = place(x, off).requires_grad_(True)

        def go():
            o = ops.segment_csr(xg, ptr.cuda(), reduce=red)
            g, = torch.autograd.grad(o, xg, gout.cuda())
            return o, g, (ops.segment_csr_arg(xg.detach(), ptr.cuda(), red) if red in ("max", "min") else None)
        # the gradients are fresh, aligned tensors: a misaligned source sends only the forward to the scalar kernel
        routed = not (off and "bwd" in case["kernel"])
        (o, g, arg_out), names = record(go, (case["kernel"],) if routed else ())
        ran |= names
        x64 = x.double().requires_grad_(True)
        ref = S_segment_csr(x64, ptr, reduce=red)
        gref, = torch.autograd.grad(ref, x64, gout.double())
        ref = ref.detach()
        if red in ("max", "min"):
            assert torch.equal(o.cpu().double(), ref), f"segment_csr {red} values"
            assert torch.equal(g.cpu().double(), gref), f"segment_csr {red} gradient"
            rv, ra = S_segment_csr_arg(x.double(), ptr, reduce=red)
            assert torch.equal(arg_out[0].cpu().double(), rv), "segment_csr_arg values"
            assert torch.equal(arg_out[1].cpu(), ra), "segment_csr_arg: first row of ties"
        else:
            check(f"segment_csr {red}", o, ref, _sum_bound(dt, x.double().abs(), ptr, ref, mean=red == "mean"))
            check(f"segment_csr {red} gradient", g, gref, (U_S[dt] + K_ERR * U32) * gref.abs() + TINY[dt])
    assert_ran(case["kernel"], ran)


def run_gather(case):
    from deepviewagg_b200 import ops
    dt = case["dtype"]
    gen = torch.Generator().manual_seed(21)
    ptr = ptr_of(segment_counts(gen, 300))
    N, V, ran = ptr.numel() - 1, int(ptr[-1]), set()
    for K, off in _seg_confs(dt, case["vec"]):
        src = _seg_values(gen, dt, N, K)
        gout = torch.randn(V, K, generator=gen).to(DTYPES[dt])
        sg = place(src, off).requires_grad_(True)

        def go():
            o = ops.gather_csr(sg, ptr.cuda(), n_items=V)
            return o, torch.autograd.grad(o, sg, gout.cuda())[0]
        (o, g), names = record(go, (case["kernel"],))
        ran |= names
        assert torch.equal(o.cpu().double(), O.gather_csr(src.double(), ptr)), "gather_csr is a copy"
        gref = S_segment_csr(gout.double(), ptr, reduce="sum")
        check("gather_csr gradient", g, gref, _sum_bound(dt, gout.double().abs(), ptr, gref))
    assert_ran(case["kernel"], ran)


def run_softmax(case):
    from deepviewagg_b200 import ops
    dt = case["dtype"]
    confs = [(8, 0)] if case["vec"] == 4 else ([(7, 0), (8, 1)] if dt == "f32" else [(4, 0), (7, 1)])
    gen = torch.Generator().manual_seed(31)
    ran = set()
    for K, off in confs:
        counts = segment_counts(gen, 300)
        ptr = ptr_of(counts)
        V = int(ptr[-1])
        dense = O.dense_index(ptr)
        x = (torch.randn(V, K, generator=gen) * 2).to(DTYPES[dt])
        x[::5] += 500                                        # max-centring matters
        for scaling in (False, True):
            gout = torch.randn(V, K, generator=gen).to(DTYPES[dt])
            xg = place(x, off).requires_grad_(True)

            def go():
                o = ops.segment_softmax_csr(xg, ptr.cuda(), scaling=scaling)
                return o, torch.autograd.grad(o, xg, gout.cuda())[0]
            (o, g), names = record(go, (case["kernel"],))
            ran |= names
            x64 = x.double().requires_grad_(True)
            ref = O.segment_softmax_csr(x64, ptr, scaling=scaling)
            n = counts[dense].double().view(-1, 1)
            s = n.sqrt() if scaling else torch.ones_like(n)
            r = n + (x.double() - S_segment_csr(x.double(), ptr, reduce="max")[dense]).abs() / s + 2
            check(f"softmax(scaling={scaling})", o, ref.detach(),
                  U_S[dt] * ref.detach().abs() + K_ERR * U32 * r * ref.detach() + TINY[dt])
            # the backward reads the stored probabilities a: against the chain rule through a, then through
            # the float64 probabilities, whose difference from a enters as a relative error da
            a, god = o.cpu().double(), gout.double()
            spread = a * (god.abs() + S_segment_csr(a * god.abs(), ptr, reduce="sum")[dense]) / s
            gref = a * (god - S_segment_csr(a * god, ptr, reduce="sum")[dense]) / s
            check(f"softmax gradient(scaling={scaling})", g, gref,
                  U_S[dt] * gref.abs() + K_ERR * U32 * (n + 2) * spread + TINY[dt])
            gref64, = torch.autograd.grad(ref, x64, god)
            da = U_S[dt] + K_ERR * U32 * r
            check(f"softmax gradient vs float64 (scaling={scaling})", g, gref64,
                  U_S[dt] * gref64.abs() + (2 * da + K_ERR * U32 * (n + 2)) * spread + TINY[dt])
    assert_ran(case["kernel"], ran)


def run_pick(case):
    from deepviewagg_b200 import ops
    dt = case["dtype"]
    gen = torch.Generator().manual_seed(41)
    ptr = ptr_of(segment_counts(gen, 300))
    V, ran = int(ptr[-1]), set()
    xmap = torch.randn(V, 3, generator=gen)
    xmap[1::4, 1] = xmap[0::4, 1][:xmap[1::4].shape[0]]       # ties in the picked feature
    for K, off in _seg_confs(dt, case["vec"]):
        x = _seg_values(gen, dt, V, K)
        for mode in ("max", "min"):
            gout = torch.randn(ptr.numel() - 1, K, generator=gen).to(DTYPES[dt])
            xg = place(x, off).requires_grad_(True)

            def go():
                o = ops.heuristic_pool(xg, xmap.cuda(), ptr.cuda(), 1, mode=mode)
                return o, torch.autograd.grad(o, xg, gout.cuda())[0]
            (o, g), names = record(go, (case["kernel"],))
            ran |= names
            x64 = x.double().requires_grad_(True)
            ref = O.heuristic_pool(x64, xmap.double(), ptr, feat=1, mode=mode)
            gref, = torch.autograd.grad(ref, x64, gout.double())
            assert torch.equal(o.cpu().double(), ref.detach()), f"heuristic_pool {mode}"
            assert torch.equal(g.cpu().double(), gref), f"heuristic_pool {mode} gradient"
    assert_ran(case["kernel"], ran)


def run_scatter(case):
    from deepviewagg_b200 import ops
    dt = case["dtype"]
    gen = torch.Generator().manual_seed(51)
    ran = set()
    for C, off in _seg_confs(dt, case["vec"]):
        V, R = 3000, 700
        src = torch.randn(V, C, generator=gen).to(DTYPES[dt])
        idx = torch.randint(0, R + 1, (V,), generator=gen)    # duplicates; R: no row, skipped
        dst, names = record(lambda: ops._scatter_add_rows(place(src, off), idx.cuda(), R), (case["kernel"],))
        ran |= names
        keep = idx < R
        ref = torch.zeros(R, C, dtype=torch.float64).index_add_(0, idx[keep], src.double()[keep])
        absref = torch.zeros(R, C, dtype=torch.float64).index_add_(0, idx[keep], src.double().abs()[keep])
        cnt = torch.bincount(idx[keep], minlength=R).double().view(-1, 1)
        check("scatter_add_rows", dst, ref, K_ERR * U32 * cnt * absref + 2.0 ** -126)
    assert_ran(case["kernel"], ran)


def run_qk(case):
    from deepviewagg_b200 import ops
    gen = torch.Generator().manual_seed(61)
    ran = set()
    for G, D, off in case["shapes"]:
        counts = segment_counts(gen, 300)
        ptr = ptr_of(counts)
        N, V = counts.numel(), int(ptr[-1])
        k, q = torch.randn(V, G * D, generator=gen), torch.randn(N, G * D, generator=gen)
        gc = torch.randn(V, G, generator=gen)
        kg, qg = place(k, off).requires_grad_(True), place(q, off).requires_grad_(True)

        def go():
            c = ops.qk_scores(kg, qg, ptr.cuda(), G, True)
            return (c,) + torch.autograd.grad(c, [kg, qg], gc.cuda())
        (c, gk, gq), names = record(go, (case["kernel"],))
        ran |= names
        k64, q64 = k.double().requires_grad_(True), q.double().requires_grad_(True)
        ref = O.qk_compatibilities(k64, q64, ptr, G, True)
        rk, rq = torch.autograd.grad(ref, [k64, q64], gc.double())
        scale = D ** -0.5
        absdot = (k.double().abs() * q.double()[O.dense_index(ptr)].abs()).view(V, G, D).sum(2) * scale
        check("qk compat", c, ref.detach(), K_ERR * U32 * (D + 2) * absdot + 2.0 ** -126)
        check("qk grad keys", gk, rk, K_ERR * U32 * rk.abs() + 2.0 ** -126)
        absg = S_segment_csr((gc.double().abs() * scale).repeat_interleave(D, 1) * k.double().abs(), ptr, reduce="sum")
        check("qk grad queries", gq, rq, K_ERR * U32 * (counts.double().view(-1, 1) + 2) * absg + 2.0 ** -126)
    assert_ran(case["kernel"], ran)


RUNNERS = dict(segment_csr=run_segment_csr, gather_csr=run_gather, softmax=run_softmax, pick=run_pick,
               scatter=run_scatter, qk=run_qk)


def test_every_instantiation_launched(va_path):
    """The union of the kernels recorded by all cases is exactly the case table (cases not run yet in this
    session, e.g. under -k, are run here)."""
    for case in CASES:
        if case["kernel"] not in SEEN:
            try:
                _run_case(case, va_path)
            except AssertionError:
                pass
    table = set(CASE_IDS)
    assert SEEN == table, {"never launched": sorted(table - SEEN), "launched without a case": sorted(SEEN - table)}
