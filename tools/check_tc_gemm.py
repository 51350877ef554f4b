"""Correctness + timing of the hand-written wgmma rows kernel (dva_tc_rows_gemm) vs fp64 torch,
next to the library paths it replaces.  python tools/check_tc_gemm.py [--quick] [--out FILE]"""
import ctypes
import json
import sys
import os

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from deepviewagg_b200 import _lib

lib = ctypes.CDLL(_lib.LIB_PATH)
lib.dva_tc_rows_workspace_bytes.restype = ctypes.c_size_t
lib.dva_tc_rows_workspace_bytes.argtypes = [ctypes.c_int64, ctypes.c_int64]
lib.dva_tc_rows_gemm.restype = ctypes.c_int
lib.dva_tc_rows_gemm.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int64] * 6 + [ctypes.c_int, ctypes.c_void_p,
                                 ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
lib.dva_last_error.restype = ctypes.c_char_p


def run(x, w, transpose, stats=False):
    M, K = x.shape
    N = w.shape[1] if transpose else w.shape[0]
    out = torch.empty(M, N, device="cuda")
    ws = torch.empty(lib.dva_tc_rows_workspace_bytes(N, K), dtype=torch.uint8, device="cuda")
    st = torch.zeros(132, 3, 128, device="cuda") if stats else None
    nct = ctypes.c_int(0)
    rc = lib.dva_tc_rows_gemm(x.data_ptr(), w.data_ptr(), out.data_ptr(), M, N, K, K, w.shape[1], N, int(transpose),
                              st.data_ptr() if stats else None, ctypes.byref(nct), ws.data_ptr(), ws.numel(),
                              torch.cuda.current_stream().cuda_stream)
    if rc != 0:
        raise RuntimeError(f"rc={rc}: {lib.dva_last_error().decode()}")
    return out, st, nct.value


def timeit(fn, n=10):
    fn(); torch.cuda.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    quick = "--quick" in sys.argv
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else ""
    torch.manual_seed(0)
    res = []
    shapes = [(1000, 128, 128), (128, 32, 128), (129, 128, 64), (5000, 64, 32), (40000, 96, 200), (30000, 256, 256),
              (20000, 512, 512), (777, 40, 36), (100000, 128, 128)]
    for (M, K, N) in shapes:
        for tr in (0, 1):
            x = torch.randn(M, K, device="cuda")
            w = torch.randn(K, N, device="cuda") if tr else torch.randn(N, K, device="cuda")
            out, st, nct = run(x, w, tr, stats=N <= 128)
            ref = x.double() @ (w.double() if tr else w.double().t())
            err = float((out.double() - ref).abs().max() / ref.abs().max())
            serr = None
            if st is not None:       # the fused statistics entry point: mean / invstd vs fp64
                mean = torch.empty(N, device="cuda"); invstd = torch.empty(N, device="cuda")
                if not tr and N % 4 == 0 and _lib.load().dva_linear_bnstats_supported(M, N, K):
                    l2 = _lib.load()
                    wsb = int(l2.dva_linear_bnstats_workspace_bytes(N, K))
                    ws2 = torch.empty(wsb, dtype=torch.uint8, device="cuda")
                    z2 = torch.empty(M, N, device="cuda")
                    _lib.check(l2.dva_linear_bnstats_fwd(x.data_ptr(), w.data_ptr(), z2.data_ptr(), M, N, K, 1e-5, 0.1,
                                                         mean.data_ptr(), invstd.data_ptr(), None, None, ws2.data_ptr(), wsb,
                                                         torch.cuda.current_stream().cuda_stream), "bnstats")
                    rm = ref.mean(0); rv = ref.var(0, unbiased=False)
                    serr = max(float((mean.double() - rm).abs().max() / rm.abs().max().clamp(min=1e-3)),
                               float((invstd.double() - (rv + 1e-5).rsqrt()).abs().max() * rv.sqrt().max()))
            res.append(dict(M=M, K=K, N=N, transpose=tr, rel_err=err, stats_err=serr))
            print(res[-1], flush=True)
    # dW through the public entry point (layout 2): D[N, K] = dZ[M, N]^T . X[M, K]
    from deepviewagg_b200 import ops
    for (M, K, N) in [(1000, 128, 128), (33, 128, 128), (5000, 128, 32), (70000, 96, 200), (30000, 256, 256),
                      (20000, 512, 512), (300000, 128, 128), (4000, 36, 132)]:
        x = torch.randn(M, K, device="cuda")
        dz = torch.randn(M, N, device="cuda")
        out = ops._tc_gemm(dz, x, 2, K)
        ref = dz.double().t() @ x.double()
        res.append(dict(dW=True, M=M, K=K, N=N, rel_err=float((out.double() - ref).abs().max() / ref.abs().max())))
        print(res[-1], flush=True)
    if not quick:
        for (M, K, N) in [(8_000_000, 128, 128), (1_280_000, 64, 128), (1_280_000, 64, 64), (1_600_000, 128, 128), (1_000_000, 512, 512)]:
            x = torch.randn(M, K, device="cuda")
            dz = torch.randn(M, N, device="cuda")
            ms = timeit(lambda: ops._tc_gemm(dz, x, 2, K))
            floor = 4.0 * M * (K + N) / 3350e9 * 1e3          # H100 SXM data-sheet HBM3 bandwidth
            res.append(dict(dW=True, M=M, K=K, N=N, ms=ms, hbm_floor_ms=floor, frac_of_floor=floor / ms))
            print(res[-1], flush=True)
            del x, dz
        for (M, K, N) in [(8_000_000, 128, 128), (8_000_000, 64, 64), (1_280_000, 64, 64), (2_000_000, 256, 256),
                          (1_000_000, 512, 512), (4_000_000, 128, 32)]:
            x = torch.randn(M, K, device="cuda")
            w = torch.randn(N, K, device="cuda")
            ms = timeit(lambda: run(x, w, 0))
            ms_s = timeit(lambda: run(x, w, 0, stats=True)) if N <= 128 else None
            floor = 4.0 * M * (K + N) / 3350e9 * 1e3          # H100 SXM data-sheet HBM3 bandwidth
            torch.backends.cuda.matmul.allow_tf32 = True
            ms_tf32 = timeit(lambda: x @ w.t())
            torch.backends.cuda.matmul.allow_tf32 = False
            res.append(dict(M=M, K=K, N=N, ms=ms, ms_with_stats=ms_s, hbm_floor_ms=floor, frac_of_floor=floor / ms,
                            cublas_tf32_ms=ms_tf32, tflops_3xtf32=6.0 * M * K * N / ms / 1e9))
            print(res[-1], flush=True)
            del x, w
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
