#!/usr/bin/env python
"""Time the fused view-attention backward alone at bench.py's flagship shape, where it runs the lane-per-view
kernel (va_lane_bwd_kernel, view_attention_lane.cu): 1 M points x 32 views x 128 ch fp32, rows gathered through a
random permutation, gating and group scaling on, the same seeded inputs as bench.py.

    python tools/bench_lane_bwd.py [--launches 100] [--warmup 10] [--points N --views V --channels C]

Prints one JSON line: the card and its power limit; the backward call's time (device events around --launches
back-to-back calls, so it includes the range-queue reset and the gate-gradient reduce); the kernels of one call
with their device times, grid and CTAs per SM, from a separate torch.profiler run.  The launcher sizes the grid
as 132 SMs x the CTAs per SM cudaOccupancyMaxActiveBlocksPerMultiprocessor allows, so grid / 132 is the
occupancy it chose.  DVA_B200_LIB=<path> times another build of the library.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import algorithmic_bytes, gpu_identity  # noqa: E402


def profile_one_call(plan):
    """Device time, grid and CTAs per SM of each kernel of one backward call."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        plan.backward_device()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    kernels = []
    for e in events:
        if e.get("cat") not in ("kernel", "gpu_memset"):
            continue
        a = e.get("args", {})
        kernels.append({"name": e["name"][:120], "us": e.get("dur"), "grid": a.get("grid"),
                        "block": a.get("block"), "blocks_per_sm": a.get("blocks per SM"),
                        "registers": a.get("registers per thread"), "smem": a.get("shared memory")})
    return kernels


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--points", type=int, default=1_000_000)
    p.add_argument("--views", type=int, default=32)
    p.add_argument("--channels", type=int, default=128)
    p.add_argument("--launches", type=int, default=100)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--label", default="")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lane_bwd.py needs a CUDA device")
    if args.launches < 50:
        raise SystemExit("--launches: at least 50")
    from deepviewagg_b200 import _lib
    from deepviewagg_b200.host_api import ViewAttentionHostPlan

    dev = torch.device("cuda", 0)
    N, v, C, G = args.points, args.views, args.channels, 4
    gen = torch.Generator(device=dev).manual_seed(1234)           # bench.py's inputs (rank 0, uniform counts)
    V = N * v
    plan = ViewAttentionHostPlan(N, V, V, C, G, dtype=torch.float32, idx_dtype=torch.int32, gating=True,
                                 group_scaling=True, device=dev)
    plan.ptr.copy_(torch.arange(0, V + 1, v, dtype=torch.long, device=dev))
    plan.x.normal_(generator=gen)
    plan.idx.copy_(torch.randperm(V, device=dev, generator=gen).int())
    plan.compat.normal_(generator=gen)
    plan.gate[0].fill_(1.0)
    plan.gate[1].fill_(0.0)
    plan.gout.normal_(generator=gen)
    plan.forward_device()                                          # the saved statistics the backward reads
    for _ in range(args.warmup):
        plan.backward_device()
    torch.cuda.synchronize()

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.launches + 1)]
    ev[0].record()
    for k in range(args.launches):
        plan.backward_device()
        ev[k + 1].record()
    torch.cuda.synchronize()
    per = [ev[k].elapsed_time(ev[k + 1]) for k in range(args.launches)]
    mean_ms = ev[0].elapsed_time(ev[-1]) / args.launches
    kernels = profile_one_call(plan)
    lane = [k for k in kernels if "va_lane_bwd_kernel" in k["name"]]
    props = torch.cuda.get_device_properties(dev)
    b_bwd = algorithmic_bytes(N, V, C, G, 4)[1]
    print(json.dumps({
        "label": args.label, "lib": _lib.LIB_PATH, "gpu": gpu_identity(0), "sms": props.multi_processor_count,
        "shape": f"{N} points x {v} views x {C} ch fp32, idx=randperm, gating, group_scaling",
        "launches": args.launches, "bwd_ms_mean": mean_ms, "bwd_ms_min": min(per),
        "bwd_ms_median": statistics.median(per), "bwd_ms_max": max(per),
        "achieved_gbs": b_bwd / (mean_ms * 1e-3) / 1e9,
        "lane_ctas_per_sm": (lane[0]["grid"][0] / props.multi_processor_count) if lane and lane[0]["grid"] else None,
        "kernels": kernels}))


if __name__ == "__main__":
    main()
