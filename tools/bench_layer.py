#!/usr/bin/env python
"""One MLP layer  a = LeakyReLU(BN(x W^T))  forward + backward at the row counts of the shipped configs:
fused (one autograd node, dva_mlp_layer_bwd) against the unfused chain (DVA_MLP_LAYER_FUSED=0 route).
    python tools/bench_layer.py [--rows 1281650] [--out FILE]"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_281_650)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    from deepviewagg_b200 import ops
    M = args.rows
    lines = []
    for K, N, need_dx in [(8, 32, False), (32, 32, True), (64, 32, True), (64, 64, True), (128, 128, True)]:
        x = torch.randn(M, K, device="cuda").requires_grad_(need_dx)
        w = (torch.randn(N, K, device="cuda") / K ** 0.5).requires_grad_(True)
        bn = torch.nn.BatchNorm1d(N).cuda()
        g = torch.randn(M, N, device="cuda")
        res = {"rows": M, "K": K, "N": N, "dx": need_dx}
        for fused in (1, 0):
            ops._MLP_LAYER_FUSED["on"] = bool(fused)
            holder = {}

            def fwd():
                holder["y"] = ops.linear_bn_act(x, w, bn, negative_slope=0.2)

            def bwd():
                torch.autograd.grad(holder["y"], ([x] if need_dx else []) + [w, bn.weight, bn.bias], g, retain_graph=True)
            tf = timeit(fwd)
            fwd()
            tb = timeit(bwd)
            key = "fused" if fused else "unfused"
            res[key + "_node"] = type(holder["y"].grad_fn).__name__
            res[key + "_fwd_ms"], res[key + "_bwd_ms"] = round(tf, 4), round(tb, 4)
        ops._MLP_LAYER_FUSED["on"] = True
        # algorithmic bytes: fwd reads x, writes z, reads z, writes a; bwd (fused) reads dA, z twice, x, writes dX
        res["bwd_floor_ms"] = round(4.0 * M * (4 * N + K + (K if need_dx else 0)) / 3350e9 * 1e3, 4)
        print(json.dumps(res), flush=True)
        lines.append(res)
        del x, w, g
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
