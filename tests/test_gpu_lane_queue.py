"""The lane-per-view backward's range queue (view_attention_lane.cu): warps take ranges of points from a counter, and
the gate-gradient partials are written per range and summed in range order.  Which warp takes which range must not
change a result: grad_x and grad_compat are bit for bit those of the static range split the queue replaced (SHA-256
of its outputs on the same seeded inputs), and grad_gate is bitwise reproducible run to run and within fp32
reordering of the static split's.  The shapes hold ragged counts, unseen points, points of more than 32 views (the
chunked path), more ranges than the largest grid has warps, in a count that is not a multiple of it, and 9 M points
holding one view, where a range is as long as it may be."""
import hashlib

import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_WARPS = 132 * 5 * 4          # the lane launcher's largest grid: 132 SMs x 5 CTAs (rows < 512 bytes) x 4 warps

# name: dtype, channels, points, mean views (0: one view in all), idx (a permutation scattered through, or none)
CASES = {
    "f32_c128_perm": (torch.float32, 128, 4000, 12.0, "perm"),        # LPR 32, the instantiation bench.py runs
    "bf16_c256_perm": (torch.bfloat16, 256, 1500, 9.0, "perm"),       # LPR 32, 2-byte storage
    "f32_c16_many_ranges": (torch.float32, 16, 120_000, 12.0, None),  # LPR 4, more ranges than warps
    "f32_c16_one_view": (torch.float32, 16, 9_000_000, 0.0, "perm"),  # 256 N / V beyond 32 bits
}

# the static range split's results on these inputs (H100): sha256(grad_x), sha256(grad_compat), grad_gate
# [dw0..3, db0..3]
EXPECTED = {
    "f32_c128_perm": ("8249ee4f392ea8db23041b1205f4ad970aadc41234622ff7f25bbfae77cbb59a",
                      "c8b3163818131b51713ab97f8eb5d8a3d8cfb4a9f05920bfdd931d9d25c32575",
                      [16.14115333557129, -22.602645874023438, -15.638029098510742, -46.414398193359375,
                       30.670917510986328, -24.92670249938965, -9.01188850402832, -54.521583557128906]),
    "bf16_c256_perm": ("20c0818832316c23b592771dede179de188b9d457bf656b1ff2152a0c3905176",
                       "e5283885eb95cc942cc387d33995fb658f8d845b9e5ca7094e0483a4104ae82f",
                       [0.8346576690673828, 24.727371215820312, 10.097410202026367, -55.94593048095703,
                        29.876266479492188, 32.63653564453125, 20.469562530517578, -98.95521545410156]),
    "f32_c16_many_ranges": ("ebcf93f27359b05d84b3dfc36721cb20a9aec408b3687ae4b1fd161cf1945f2f",
                            "25ced4fbe9af4b0a154b3a5ae4a4b2db27e65b7a291a760b87525764b57a044e",
                            [95.60971069335938, 29.335012435913086, -24.252073287963867, -41.360755920410156,
                             116.31137084960938, 13.026378631591797, -16.715023040771484, -18.429630279541016]),
    "f32_c16_one_view": ("294096e9bdda7e6a57d7bd5876fa93a4097563b9f58da09f6391b7dc6b3a8103",
                         "6808849af8bcb358362e6d66428ffbd2550b675d40a2713cc0e00b655cbf07c1",
                         [-0.19421622157096863, -0.7410178184509277, 0.0, 0.0,
                          -0.22404201328754425, -0.63026362657547, 0.0, 0.0]),
}
# grad_gate against the static split's, relative to its largest element: the two sum the same per-point terms in
# another order, 3.1e-7 apart at most here (the streaming kernel's order: 4.6e-7)
GATE_TOL = 1e-5


def lane_ranges(N, V):
    """Python copy of lane_range_points (view_attention.cuh): (points per range, number of ranges)."""
    pr = max(min(-(-256 * N // max(V, 1)), 8192), -(-N // (1 << 17)), 1)
    return pr, -(-N // pr)


def inputs(name):
    dtype, C, N, mean, idx_kind = CASES[name]
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    if mean == 0:
        counts = torch.zeros(N, dtype=torch.long)
        counts[N // 3] = 1
    else:
        counts = torch.poisson(torch.full((N,), mean), generator=gen).clamp(0, 32).long()
        counts[torch.rand(N, generator=gen) < 0.1] = 0                               # unseen points
        counts[torch.randint(0, N, (max(N // 200, 3),), generator=gen)] = \
            torch.randint(33, 100, (max(N // 200, 3),), generator=gen)              # chunked path
    ptr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)])
    V = int(ptr[-1])
    return dict(
        x=torch.randn(V, C, generator=gen).to(dtype), compat=torch.randn(V, 4, generator=gen), ptr=ptr,
        idx=torch.randperm(V, generator=gen).int() if idx_kind == "perm" else None,
        gw=torch.tensor([[1.1, 0.9, -0.4, 0.7]]), gb=torch.tensor([[0.05, -0.1, 0.3, 0.0]]),
        gout=torch.randn(N, C, generator=gen).to(dtype))


def run(inp):
    """One forward + backward on the lane backward: (grad_x, grad_compat, grad_gate [8])."""
    from deepviewagg_b200 import ops
    x = inp["x"].cuda().requires_grad_(True)
    c = inp["compat"].cuda().requires_grad_(True)
    gw = inp["gw"].cuda().requires_grad_(True)
    gb = inp["gb"].cuda().requires_grad_(True)
    idx = inp["idx"].cuda() if inp["idx"] is not None else None
    out, _, _ = ops.view_attention(x, c, inp["ptr"].cuda(), 4, idx=idx, gate_weight=gw, gate_bias=gb,
                                   group_scaling=True, idx_is_permutation=idx is not None)
    gx, gc, ggw, ggb = torch.autograd.grad(out, [x, c, gw, gb], inp["gout"].cuda())
    torch.cuda.synchronize()
    return gx, gc, torch.cat([ggw.view(-1), ggb.view(-1)])


def digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


@pytest.fixture
def lane_path():
    from deepviewagg_b200 import _lib
    lib = _lib.load()
    assert lib.dva_view_attention_set_path(3) == 0
    yield
    assert lib.dva_view_attention_set_path(0) == 0


@pytest.mark.parametrize("name", list(CASES))
def test_lane_queue_results(name, lane_path):
    inp = inputs(name)
    N, V = inp["ptr"].numel() - 1, int(inp["ptr"][-1])
    pr, n_ranges = lane_ranges(N, V)
    if name.endswith("many_ranges"):
        assert n_ranges > MAX_WARPS and n_ranges % MAX_WARPS != 0, n_ranges
    if name.endswith("one_view"):
        assert 256 * N // V >= 1 << 31 and pr == 8192, pr
    gx, gc, gg = run(inp)
    gx2, gc2, gg2 = run(inp)
    assert torch.equal(gx, gx2) and torch.equal(gc, gc2) and torch.equal(gg, gg2), "not reproducible run to run"
    want_gx, want_gc, want_gg = EXPECTED[name]
    assert digest(gx) == want_gx, "grad_x differs from the static range split's"
    assert digest(gc) == want_gc, "grad_compat differs from the static range split's"
    want = torch.tensor(want_gg, dtype=torch.float64)
    err = (gg.cpu().double() - want).abs().max().item()
    assert err <= GATE_TOL * want.abs().max().item(), (err, gg.tolist(), want_gg)
