"""Micro-benchmark of the projection GEMM variants (developer tool): z = x @ W^T for x [M,K], W [N,K]."""
import sys
import torch
sys.path.insert(0, ".")
from deepviewagg_b200 import ops


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


SHAPES = ((2_000_000, 128, 128),) if "--quick" in sys.argv else ((8_000_000, 128, 128), (1_280_000, 64, 64), (8_000_000, 32, 32), (2_000_000, 512, 512))
for (M, K, N) in SHAPES:
    x = torch.randn(M, K, device="cuda")
    w = torch.randn(N, K, device="cuda") / K ** 0.5
    g = torch.randn(M, N, device="cuda")
    ref = (x[:4096].double() @ w.double().t())
    flops = 2.0 * M * K * N
    byts = 4.0 * (M * K + M * N)
    res = {}
    torch.backends.cuda.matmul.allow_tf32 = False
    res["cublas fp32"] = (timeit(lambda: x @ w.t()), (x[:4096] @ w.t()).double())
    res["cublas dW fp32"] = (timeit(lambda: g.t() @ x), None)
    torch.backends.cuda.matmul.allow_tf32 = True
    res["cublas tf32"] = (timeit(lambda: x @ w.t()), (x[:4096] @ w.t()).double())
    res["cublas dW tf32"] = (timeit(lambda: g.t() @ x), None)
    torch.backends.cuda.matmul.allow_tf32 = False
    for mode in ("fp32", "tf32"):
        ops.set_gemm_precision(mode)
        res[f"dva wgmma {mode}"] = (timeit(lambda: ops._tc_gemm(x, w, 0, N)), ops._tc_gemm(x[:4096].contiguous(), w, 0, N).double())
        res[f"dva wgmma dX {mode}"] = (timeit(lambda: ops._tc_gemm(g, w, 1, K)), None)
        res[f"dva wgmma dW {mode}"] = (timeit(lambda: ops._tc_gemm(g, x, 2, K)), None)
    ops.set_gemm_precision("fp32")
    print(f"M={M} K={K} N={N}: {flops / 1e12:.2f} TFLOP, {byts / 1e9:.1f} GB (HBM floor {byts / 3350e9 * 1e3:.2f} ms)")
    for k, (ms, out) in res.items():
        err = "" if out is None else f" relerr {float((out - ref).abs().max() / ref.abs().max()):.1e}"
        print(f"   {k:22s} {ms:8.3f} ms  {flops / ms / 1e9:8.1f} TFLOP/s {byts / ms / 1e6:8.0f} GB/s{err}")
