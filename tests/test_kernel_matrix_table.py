"""Kernel matrix of the fused view attention, the segment primitives and qk_scores: the case table, the
inputs that route to each case, the float64 reference and its per-element error bounds.

tests/test_gpu_kernel_matrix.py runs every case on the GPU and records, by name, which kernel ran.  This file
checks, without a GPU, that
  * the case table holds exactly the instantiations compiled into libdva_b200.so (cuobjdump -symbols), so a
    new instantiation without a case fails here;
  * the per-element bounds can fail: plausible bugs injected into the float64 oracle break them.

Error bounds (u32 = 2^-24, u_s = half an ulp of the storage type, K = 8 throughout; all quantities from the
float64 reference on the exact stored inputs; n = segment length, s = sqrt(n) with group scaling else 1,
m = segment max of the scores, d_vg = |c_vg - m_g| / s, r_vg = n + d_vg + 2; gate z = w m + b, t = tanh(relu(z)),
dt = (1 - t^2)(|w m| + |b|) + |t| the absolute error of t in units of u32; without gating t = 1, dt = 0):
  out_ic    <= u_s |ref| + K u32 (|t_g| sum_v r_vg a_vg |x_vc| + dt_g sum_v a_vg |x_vc|)
  att_vg    <= K u32 r_vg a_vg
  grad_x_rc <= u_s |ref| + sum_{v -> r} |a_vg gout_c| (K u32 (r_vg |t_g| + dt_g + cnt_r) + u_s |t_g|)
  grad_compat_vg <= K u32 a_vg ((r_vg + C_g) P_vg |t| + Qr_g |t| + dt (P_vg + Q_g)) / s
                    + [v = first arg-max] |w_g| e_g
     with P_vg = sum_{c in g} |gout_c x_vc|, Q_g = sum_v a_vg P_vg, Qr_g = sum_v a_vg (r_vg + C_g) P_vg,
     e_g = K u32 ((1 - t^2) Qr_g + 2 |t| dt |dL/dt|) where the gate is open, plus |dL/dt| where |z| is within
     K u32 (|w m| + |b|) of the relu kink (either side is a correct derivative there)
  grad_w_g  <= sum_i |m_i| e_ig + K u32 L sum_i |m_i dL/dt (1 - t^2)|,   grad_b likewise without |m|,
     L = 64 + N/128 bounding the longest accumulation chain of the cross-point reduction.
Every bound also carries the storage type's smallest step (2^-126, or 2^-24 for fp16 subnormals).  Gated-out
groups (z below the kink band) and unseen points must be exactly zero.  Segment primitives: sums
u_s |ref| + K u32 n sum |x|, means the same over n, softmax K u32 (n + d) a, max / min / arg / pick and every
copy bit-equal with ties to the first row.
"""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import pooling_oracle as O
from oracle.scatter_standin import segment_csr as S_segment_csr, segment_csr_arg as S_segment_csr_arg

K_ERR = 8
U32 = 2.0 ** -24
DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
CPP = {"f32": "float", "bf16": "__nv_bfloat16", "f16": "__half"}
V16 = {"f32": 4, "bf16": 8, "f16": 8}
U_S = {"f32": 2.0 ** -24, "bf16": 2.0 ** -8, "f16": 2.0 ** -11}
TINY = {"f32": 2.0 ** -126, "bf16": 2.0 ** -126, "f16": 2.0 ** -24}
FAMILIES = ("view_attention_fwd_kernel", "view_attention_bwd_kernel", "va_ring_fwd_kernel", "va_ring_bwd_kernel",
            "va_lane_bwd_kernel", "segment_csr_fwd_kernel", "segment_csr_bwd_kernel", "gather_csr_kernel",
            "segment_softmax_fwd_kernel", "segment_softmax_bwd_kernel", "segment_softmax_fwd_v4_kernel",
            "segment_softmax_bwd_v4_kernel", "pick_rows_kernel", "scatter_add_rows_kernel",
            "qk_scores_fwd_kernel", "qk_scores_bwd_kernel", "qk_scores_fwd_vec_kernel", "qk_scores_bwd_vec_kernel")
SEG_LENGTHS = (0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257)   # a warp of views, DVA_RING_CAPV_BWD, _FWD


# ------------------------------------------------------------------------------------------------
# kernel names
# ------------------------------------------------------------------------------------------------
def parse_kernel(name, namespace="dva::"):
    """Demangled kernel name -> (family, template args), e.g.
    'void dva::view_attention_bwd_kernel<__nv_bfloat16, 1, 32, 4, 2, true>(dva::VAParams)'
    -> ('view_attention_bwd_kernel', ('__nv_bfloat16', '1', '32', '4', '2', 'true')); None outside `namespace`."""
    s = name.strip()
    if s.startswith("void "):
        s = s[5:]
    if not s.startswith(namespace):
        return None
    s = s[len(namespace):]
    cut = len(s)
    for ch in "<(":
        if ch in s:
            cut = min(cut, s.index(ch))
    family = s[:cut]
    args = ()
    if cut < len(s) and s[cut] == "<":
        args = tuple(a.strip() for a in s[cut + 1:s.index(">", cut)].split(","))
    return family, args


def kname(family, *args):
    return f"{family}<{', '.join(str(a).lower() if isinstance(a, bool) else str(a) for a in args)}>" if args \
        else family


def canonical(name, families=FAMILIES, namespace="dva::"):
    p = parse_kernel(name, namespace)
    if p is None or p[0] not in families:
        return None
    return kname(p[0], *p[1])


# ------------------------------------------------------------------------------------------------
# the case table: one entry per instantiation, with the inputs the host dispatch routes to it
# ------------------------------------------------------------------------------------------------
def _va_cases():
    cases = []

    def add(kernel, dt, C, G, path, x_off=0, c_off=0):
        cases.append(dict(kind="va", kernel=kernel, dtype=dt, C=C, G=G, path=path, x_off=x_off, c_off=c_off))

    for dt in DTYPES:
        T, V = CPP[dt], V16[dt]
        # streaming forward, VEC = 16 / sizeof(T): LPR from cv = C / VEC, CPL 2 / 4 past 32 chunks (160 chunks:
        # two channel tiles)
        for cv, lpr, cpl in ((4, 4, 1), (8, 8, 1), (16, 16, 1), (32, 32, 1), (64, 32, 2), (160, 32, 4)):
            add(kname("view_attention_fwd_kernel", T, V, lpr, cpl, 2 if cpl >= 4 else 4), dt, cv * V, 4, 1)
        # streaming backward: regular groups (a power-of-two number of chunks each); 256 chunks: two tiles
        for cv, lpr, cpl in ((4, 4, 1), (8, 8, 1), (16, 16, 1), (32, 32, 1), (64, 32, 2), (256, 32, 4)):
            add(kname("view_attention_bwd_kernel", T, V, lpr, cpl, 2 if cpl >= 4 else 4, True), dt, cv * V, 4, 1)
        # scalar kernels: a misaligned x (storage offset of one element), or chunks that straddle groups
        add(kname("view_attention_fwd_kernel", T, 1, 32, 1, 4), dt, 32, 4, 1, x_off=1, c_off=1)
        add(kname("view_attention_fwd_kernel", T, 1, 32, 4, 2), dt, 36, 4, 1)
        add(kname("view_attention_bwd_kernel", T, 1, 32, 1, 4, True), dt, 16, 8, 1)
        add(kname("view_attention_bwd_kernel", T, 1, 32, 1, 4, False), dt, 12, 4, 1)
        add(kname("view_attention_bwd_kernel", T, 1, 32, 4, 2, True), dt, 128, 4, 1, x_off=1)
        add(kname("view_attention_bwd_kernel", T, 1, 32, 4, 2, False), dt, 36, 4, 1, c_off=1)
        for cv in (4, 8, 16, 32):
            add(kname("va_ring_fwd_kernel", T, cv), dt, cv * V, 4, 2)
            add(kname("va_ring_bwd_kernel", T, cv), dt, cv * V, 4, 2)
            add(kname("va_lane_bwd_kernel", T, cv), dt, cv * V, 4, 3)
    return cases


def _seg_cases():
    cases = []
    for dt in DTYPES:
        T, V = CPP[dt], V16[dt]
        for vec in (V, 1):
            for red in range(4):        # DVA_SUM, DVA_MEAN, DVA_MAX, DVA_MIN
                for fam in ("segment_csr_fwd_kernel", "segment_csr_bwd_kernel"):
                    cases.append(dict(kind="segment_csr", kernel=kname(fam, T, vec, red), dtype=dt, vec=vec, red=red))
            cases.append(dict(kind="gather_csr", kernel=kname("gather_csr_kernel", T, vec), dtype=dt, vec=vec))
            cases.append(dict(kind="pick", kernel=kname("pick_rows_kernel", T, vec), dtype=dt, vec=vec))
            cases.append(dict(kind="scatter", kernel=kname("scatter_add_rows_kernel", T, vec), dtype=dt, vec=vec))
        for fam in ("segment_softmax_fwd_kernel", "segment_softmax_bwd_kernel"):
            cases.append(dict(kind="softmax", kernel=kname(fam, T), dtype=dt, vec=1))
    for fam in ("segment_softmax_fwd_v4_kernel", "segment_softmax_bwd_v4_kernel"):
        cases.append(dict(kind="softmax", kernel=fam, dtype="f32", vec=4))
    return cases


def _qk_cases():
    cases = []
    for G, D in ((1, 4), (2, 4), (4, 4), (4, 8), (4, 16), (8, 16)):
        for fam in ("qk_scores_fwd_vec_kernel", "qk_scores_bwd_vec_kernel"):
            cases.append(dict(kind="qk", kernel=kname(fam, G * D // 4), shapes=((G, D, 0),)))
    for fam in ("qk_scores_fwd_kernel", "qk_scores_bwd_kernel"):   # scalar: D % 4 != 0, or misaligned rows
        cases.append(dict(kind="qk", kernel=fam, shapes=((1, 3, 0), (8, 2, 0), (4, 8, 1))))
    return cases


CASES = _va_cases() + _seg_cases() + _qk_cases()
CASE_IDS = [c["kernel"] for c in CASES]


def library_kernels(lib_path, families=FAMILIES):
    """Canonical names of the listed families compiled into `lib_path` (cuobjdump -symbols | c++filt)."""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "-symbols", lib_path], capture_output=True, text=True, check=True).stdout
    mangled = [ln.split()[-1] for ln in out.splitlines() if "STT_FUNC" in ln]
    dem = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout
    return {k for k in (canonical(n, families) for n in dem.splitlines()) if k is not None}


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
VA_VARIANTS = (dict(scaling=True, gating=True, idx=None),
               dict(scaling=False, gating=False, idx="i32perm"),
               dict(scaling=True, gating=True, idx="i64dup"))


def segment_counts(gen, n_rand, mean=3.0):
    """Random short segments (15 % unseen points) with SEG_LENGTHS placed at random positions."""
    counts = torch.poisson(torch.full((n_rand,), mean), generator=gen).long()
    counts[torch.rand(n_rand, generator=gen) < 0.15] = 0
    pos = torch.randperm(n_rand + len(SEG_LENGTHS), generator=gen)[:len(SEG_LENGTHS)]
    full = torch.empty(n_rand + len(SEG_LENGTHS), dtype=torch.long)
    mask = torch.zeros(full.numel(), dtype=torch.bool)
    mask[pos] = True
    full[pos] = torch.tensor(SEG_LENGTHS)
    full[~mask] = counts
    return full


def ptr_of(counts):
    return torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)])


def va_inputs(case, variant, seed=0):
    """CPU inputs of one view-attention case: x and gout in the storage type, fp32 scores with ties and
    ~1e3-magnitude segments, a gate that closes one group everywhere and others per point."""
    dt, C, G = case["dtype"], case["C"], case["G"]
    v = VA_VARIANTS[variant]
    gen = torch.Generator().manual_seed(1000 * seed + 7 * variant + C + G)
    n_rand = int(min(4000, max(64, 1.5e6 // (4 * C))))
    counts = segment_counts(gen, n_rand)
    ptr = ptr_of(counts)
    N, V = counts.numel(), int(ptr[-1])
    compat = torch.randn(V, G, generator=gen) * 2
    for i in range(N):
        p0, n = int(ptr[i]), int(counts[i])
        if n == 0:
            continue
        if i % 5 == 0:
            compat[p0:p0 + n] += 1e3                         # max-centring matters
        if i % 7 == 0:
            compat[p0:p0 + n] = compat[p0]                   # every view tied
        elif i % 11 == 0 and n > 1:
            compat[p0 + n - 1] = compat[p0:p0 + n].max(0).values   # the arg-max tied with the last view
    idx, R = None, V
    if v["idx"] == "i32perm":
        idx = torch.randperm(V, generator=gen).int()
    elif v["idx"] == "i64dup":
        R = V + 37
        idx = torch.randint(0, R, (V,), generator=gen)
    x = torch.randn(R, C, generator=gen).to(DTYPES[dt])
    gw = gb = None
    if v["gating"]:
        gw = torch.tensor([1.0, 0.5, -0.8, 1.2] * (G // 4 + 1))[:G].view(1, G)
        gb = torch.tensor([0.3, -0.2, 0.1, -1e5] * (G // 4 + 1))[:G].view(1, G)
        if G < 4:
            gb[0, -1] = -1e5
    gout = torch.randn(N, C, generator=gen).to(DTYPES[dt])
    return dict(x=x, compat=compat, ptr=ptr, idx=idx, gw=gw, gb=gb, gout=gout, scaling=v["scaling"], G=G,
                dtype=dt, is_perm=v["idx"] == "i32perm")


# ------------------------------------------------------------------------------------------------
# float64 reference and bounds
# ------------------------------------------------------------------------------------------------
def _segsum(t, ptr):
    return S_segment_csr(t, ptr, reduce="sum")


def va_reference(inp, x=None, compat=None, ptr=None, gating=True):
    """Float64 oracle (pooling_oracle.view_attention) on the stored inputs: out, att and the gradients of
    autograd.grad(out, [x, compat, w, b], gout)."""
    x64 = (inp["x"] if x is None else x).double().requires_grad_(True)
    c64 = (inp["compat"] if compat is None else compat).double().requires_grad_(True)
    ptr = inp["ptr"] if ptr is None else ptr
    gw = gb = None
    leaves = [x64, c64]
    if gating and inp["gw"] is not None:
        gw, gb = inp["gw"].double().requires_grad_(True), inp["gb"].double().requires_grad_(True)
        leaves += [gw, gb]
    out, att = O.view_attention(x64, c64, ptr, inp["G"], idx=inp["idx"], gate_weight=gw, gate_bias=gb,
                                group_scaling=inp["scaling"])
    grads = torch.autograd.grad(out, leaves, inp["gout"].double())
    r = dict(out=out.detach(), att=att.detach(), gx=grads[0], gcompat=grads[1])
    if len(grads) > 2:
        r["gw"], r["gb"] = grads[2], grads[3]
    return r


def va_bounds(inp, ref):
    """Per-element bounds of the module docstring, float64, same shapes as the reference tensors."""
    dt, G = inp["dtype"], inp["G"]
    us, tiny, ke = U_S[dt], TINY[dt], K_ERR * U32
    ptr = inp["ptr"]
    counts = ptr[1:] - ptr[:-1]
    N, V = counts.numel(), int(ptr[-1])
    x64 = inp["x"].double()
    rows = x64 if inp["idx"] is None else x64[inp["idx"].long()]
    C = rows.shape[1]
    grp = torch.repeat_interleave(torch.arange(G), torch.tensor(O.group_sizes(C, G)))
    onehot = torch.nn.functional.one_hot(grp, G).double()                       # [C, G]
    Cg = onehot.sum(0)                                                           # [G]
    dense = O.dense_index(ptr)
    c64 = inp["compat"].double()
    m, arg = S_segment_csr_arg(c64, ptr, reduce="max")                           # [N, G]
    n_v = counts[dense].double().view(-1, 1)
    s_v = n_v.sqrt() if inp["scaling"] else torch.ones_like(n_v)
    d = (c64 - m[dense]).abs() / s_v
    a = ref["att"]
    r = n_v + d + 2
    if inp["gw"] is not None:
        w, b = inp["gw"].double().view(1, G), inp["gb"].double().view(1, G)
        z = w * m + b
        t = torch.tanh(torch.relu(z))
        dtt = (1 - t * t) * ((w * m).abs() + b.abs()) + t.abs()
        kink = z.abs() <= ke * ((w * m).abs() + b.abs())
        closed = (z < 0) & ~kink
    else:
        w = torch.zeros(1, G, dtype=torch.float64)
        t, dtt = torch.ones(N, G, dtype=torch.float64), torch.zeros(N, G, dtype=torch.float64)
        kink = closed = torch.zeros(N, G, dtype=torch.bool)
    ac, rc = a[:, grp], r[:, grp]
    tc, dtc = t[:, grp], dtt[:, grp]
    S1 = _segsum(ac * rows.abs(), ptr)
    Sr = _segsum(ac * rc * rows.abs(), ptr)
    b_out = us * ref["out"].abs() + tiny + ke * (tc.abs() * Sr + dtc * S1)
    b_att = ke * r * a + 2.0 ** -126
    # grad_x: per view, then summed onto the rows the views read
    god = inp["gout"].double()[dense]
    agt = (ac * god).abs()
    per_view = agt * (ke * (rc * tc[dense].abs() + dtc[dense]) + us * tc[dense].abs())
    R = x64.shape[0]
    if inp["idx"] is None:
        cnt = torch.ones(R, 1, dtype=torch.float64)
        b_gx = per_view
        agt_r = agt * tc[dense].abs()
    else:
        il = inp["idx"].long()
        cnt = torch.zeros(R, dtype=torch.float64).index_add_(0, il, torch.ones(V, dtype=torch.float64)).view(-1, 1)
        b_gx = torch.zeros(R, C, dtype=torch.float64).index_add_(0, il, per_view)
        agt_r = torch.zeros(R, C, dtype=torch.float64).index_add_(0, il, agt * tc[dense].abs())
    b_gx = b_gx + ke * cnt * agt_r + us * ref["gx"].abs() + tiny
    # grad_compat
    P = (god * rows).abs() @ onehot                                              # [V, G]
    Dsig = (god * rows) @ onehot
    Q = _segsum(a * P, ptr)
    Qr = _segsum(a * (r + Cg) * P, ptr)
    dLdt = _segsum(a * Dsig, ptr)
    tv, dtv = t[dense], dtt[dense]
    b_gc = ke * a * ((r + Cg) * P * tv.abs() + Qr[dense] * tv.abs() + dtv * (P + Q[dense])) / s_v + 2.0 ** -126
    res = dict(out=b_out, att=b_att, gx=b_gx, gcompat=b_gc, closed=closed)
    if inp["gw"] is not None:
        open_ = (z > 0).double()
        e = ke * ((1 - t * t) * Qr + 2 * t.abs() * dtt * dLdt.abs()) * open_ + kink.double() * dLdt.abs()
        nonempty = counts > 0
        rows_i, cols = torch.nonzero(nonempty.view(-1, 1).expand(N, G), as_tuple=True)
        b_gc = b_gc.clone()
        b_gc.index_put_((arg[rows_i, cols], cols), (w.abs().expand(N, G) * e)[rows_i, cols], accumulate=True)
        L = 64 + N // 128
        lin = (dLdt * (1 - t * t)).abs() * open_
        res["gcompat"] = b_gc
        res["gw"] = ((m.abs() * e).sum(0) + ke * L * (m.abs() * lin).sum(0)).view(1, G) + 2.0 ** -126
        res["gb"] = (e.sum(0) + ke * L * lin.sum(0)).view(1, G) + 2.0 ** -126
    return res


def violations(got, ref, bound):
    """Number of elements outside the bound (NaN counts), and a description of the worst one."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = (got - ref).abs()
    bad = ~(err <= bound)
    nbad = int(bad.sum())
    if nbad == 0:
        return 0, ""
    ratio = torch.where(bad, (err / bound).nan_to_num(float("inf")), torch.zeros_like(err))
    j = int(ratio.view(-1).argmax())
    ix = np.unravel_index(j, tuple(got.shape))
    return nbad, (f"{nbad}/{got.numel()} outside; worst at {tuple(int(i) for i in ix)}: got {got.view(-1)[j]:.9g} "
                  f"ref {ref.view(-1)[j]:.9g} bound {bound.view(-1)[j]:.3g}")


def round_to(t, dt, toward_zero=False):
    """float64 -> storage type -> float64, to nearest or toward zero."""
    if not toward_zero:
        return t.to(DTYPES[dt]).double()
    if dt == "bf16":
        bits = t.float().view(torch.int32) & ~0xFFFF
        return bits.view(torch.float32).double()
    if dt == "f16":
        a = t.numpy()
        y = a.astype(np.float16)
        away = np.abs(y.astype(np.float64)) > np.abs(a)
        y = np.where(away, np.nextafter(y, np.float16(0)), y)
        return torch.from_numpy(y.astype(np.float64))
    return t.float().double()


# ------------------------------------------------------------------------------------------------
# CPU tests
# ------------------------------------------------------------------------------------------------
def _lib_path():
    from deepviewagg_b200 import _lib
    return _lib.LIB_PATH


def test_case_table_matches_library():
    path = _lib_path()
    if not os.path.exists(path):
        pytest.fail(f"{path} is not built")
    assert len(CASE_IDS) == len(set(CASE_IDS)), "one case per instantiation"
    built = library_kernels(path)
    table = set(CASE_IDS)
    assert built == table, {"compiled without a case": sorted(built - table),
                            "case without an instantiation": sorted(table - built)}
    va = [k for k in table if k.startswith(("view_attention_", "va_"))]
    qk = [k for k in table if k.startswith("qk_scores_")]
    assert len(va) == 90 and len(qk) == 14


def test_parse_kernel_names():
    assert parse_kernel("void dva::view_attention_bwd_kernel<__nv_bfloat16, 1, 32, 4, 2, true>(dva::VAParams)") == \
        ("view_attention_bwd_kernel", ("__nv_bfloat16", "1", "32", "4", "2", "true"))
    assert canonical("dva::qk_scores_fwd_kernel(float const*, float const*, long const*, float*, long, int, int, "
                     "float)") == "qk_scores_fwd_kernel"
    assert canonical("void at::native::vectorized_elementwise_kernel<4, float>(int, float)") is None


SENS_CASES = [dict(dtype="f32", C=64, G=4), dict(dtype="bf16", C=128, G=4), dict(dtype="f16", C=32, G=4),
              dict(dtype="f32", C=36, G=4)]


@pytest.mark.parametrize("spec", SENS_CASES, ids=lambda s: f"{s['dtype']}-C{s['C']}-G{s['G']}")
def test_bounds_reject_buggy_oracles(spec):
    inp = va_inputs(spec, 0, seed=3)
    ref = va_reference(inp)
    bnd = va_bounds(inp, ref)
    dt, G, C = spec["dtype"], spec["G"], spec["C"]
    # the correct result, rounded to the storage type, is inside its bounds
    assert violations(round_to(ref["out"], dt), ref["out"], bnd["out"])[0] == 0
    ptr, counts = inp["ptr"], inp["ptr"][1:] - inp["ptr"][:-1]
    rejected = {}
    # 1. the last view of every segment dropped
    keep = torch.ones(int(ptr[-1]), dtype=torch.bool)
    keep[(ptr[1:] - 1)[counts > 0]] = False
    out1 = va_reference(dict(inp, idx=None), x=inp["x"][keep], compat=inp["compat"][keep],
                        ptr=ptr_of(torch.clamp(counts - 1, min=0)))["out"]
    rejected["drop last view"] = violations(round_to(out1, dt), ref["out"], bnd["out"])[0]
    # 2. one 16-byte chunk read one channel late
    vec = V16[dt]
    x2 = inp["x"].clone()
    x2[:, vec:2 * vec] = inp["x"][:, vec + 1:2 * vec + 1]
    rejected["chunk shifted"] = violations(round_to(va_reference(inp, x=x2)["out"], dt), ref["out"], bnd["out"])[0]
    # 3. the gate of group 0 skipped
    ungated = va_reference(inp, gating=False)["out"]
    grp = torch.repeat_interleave(torch.arange(G), torch.tensor(O.group_sizes(C, G)))
    out3 = ref["out"].clone()
    out3[:, grp == 0] = ungated[:, grp == 0]
    rejected["gate skipped"] = violations(round_to(out3, dt), ref["out"], bnd["out"])[0]
    # 4. centred scores divided by n instead of sqrt(n)
    n_v = counts[O.dense_index(ptr)].double().clamp(min=1).sqrt().float().view(-1, 1)
    r4 = va_reference(inp, compat=inp["compat"] / n_v)
    rejected["scaled by n"] = violations(r4["att"], ref["att"], bnd["att"])[0]
    # 5. half outputs rounded toward zero
    if dt != "f32":
        rejected["round toward zero"] = violations(round_to(ref["out"], dt, toward_zero=True), ref["out"],
                                                   bnd["out"])[0]
    assert all(v > 0 for v in rejected.values()), rejected
