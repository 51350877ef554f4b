"""Segmentation evaluation timings (ops.confusion_update, ops.vote, ops.full_res_predict) against the reference's
host path and against torch on the GPU.  One JSON line per case on stdout and in --out; the card name and its power
limit are read in the same run.  Times are CUDA-event medians after warm-up."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepviewagg_b200 import ops  # noqa: E402
from deepviewagg_b200._lib import launch  # noqa: E402
from deepviewagg_b200.core.multimodal.mapping import knn_query  # noqa: E402

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def gpu_ms(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        t.append(a.elapsed_time(b))
    return float(np.median(t))


def host_ms(fn, reps=5):
    fn()
    t = []
    for _ in range(reps):
        torch.cuda.synchronize()
        s = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append((time.perf_counter() - s) * 1e3)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    rows = []
    gpu = card()

    def emit(**r):
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)

    # per-batch update at the S3DIS step shape
    n, K = 383_000, 13
    labels = torch.randint(0, K, (n,), generator=g, device=dev)
    labels[torch.rand(n, generator=g, device=dev) < 0.1] = -1
    cm = torch.zeros(K, K, dtype=torch.int64, device=dev)
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        s = torch.randn(n, K, generator=g, device=dev).to(dt)
        ours = gpu_ms(lambda: ops.confusion_update(cm, s, labels, ignore_label=-1))

        def torch_gpu():
            keep = labels != -1
            return torch.bincount(K * labels[keep] + s[keep].argmax(1), minlength=K * K)

        def reference():
            lab = labels.cpu().numpy()
            m = lab != -1
            out = s.float().cpu().numpy()[m] if s.dtype != torch.float32 else s.cpu().numpy()[m]
            return np.bincount(K * lab[m] + np.argmax(out, 1), minlength=K * K)
        nbytes = n * K * s.element_size() + 8 * n
        emit(case="confusion_update", n=n, K=K, dtype=str(dt).split(".")[-1], ms=ours, torch_gpu_ms=gpu_ms(torch_gpu),
             reference_host_ms=host_ms(reference), hbm_share=nbytes / (ours * 1e-3) / HBM)

    # vote accumulation: 383 k rows into a 10 M-point table
    N = 10_000_000
    votes = torch.zeros(N, K, device=dev)
    counts = torch.zeros(N, dtype=torch.int32, device=dev)
    stamp = torch.full((N,), -1, dtype=torch.int32, device=dev)
    ids = torch.randperm(N, generator=g, device=dev)[:n]
    out = torch.randn(n, K, generator=g, device=dev)
    ours = gpu_ms(lambda: ops.vote(votes, counts, stamp, ids, out))

    def index_put():
        votes[ids] += out
        counts[ids] += 1
    emit(case="vote", n=n, N=N, K=K, ms=ours, torch_gpu_ms=gpu_ms(index_put))

    # full resolution: 10 M points with ~9 M voted, and a window with a 40 % unvoted share
    for name, NN, share, mode in (("area", 10_000_000, 0.9, "interpolate"), ("window", 3_000_000, 0.6, "own_votes")):
        pos = torch.rand(NN, 3, generator=g, device=dev) * torch.tensor([50.0, 50.0, 5.0], device=dev)
        cnt = (torch.rand(NN, generator=g, device=dev) < share).int()
        v = torch.randn(NN, K, generator=g, device=dev) * cnt[:, None]
        y = torch.randint(0, K, (NN,), generator=g, device=dev)
        c = torch.zeros(K, K, dtype=torch.int64, device=dev)
        ours = gpu_ms(lambda: ops.full_res_predict(v, cnt, pos, labels=y, cm=c, mode=mode), reps=5, warm=1)
        voted = torch.nonzero(cnt > 0).squeeze(1)
        q = torch.nonzero(cnt == 0).squeeze(1) if mode == "own_votes" else torch.arange(NN, device=dev)
        nbr = knn_query(pos[q], pos[voted], 1).squeeze(1)
        knn = gpu_ms(lambda: knn_query(pos[q], pos[voted], 1), reps=5, warm=1)
        full_nbr = torch.zeros(NN, dtype=torch.int64, device=dev)
        full_nbr[q] = nbr
        qall = torch.arange(NN, device=dev)
        pred = torch.empty(NN, dtype=torch.int64, device=dev)
        st = ops.eval_status(dev)
        fused = gpu_ms(lambda: launch("dva_eval_nn_vote", dev, v, cnt, pos, NN, K, voted, voted.numel(), qall, full_nbr,
                                      NN, ops._NN_MODES[mode], y, 0, 0, pred, c, st), reps=5, warm=1)

        def chain():
            xv = v[voted]
            diff = pos[voted][nbr] - pos[q]
            d2 = (diff * diff).sum(-1, keepdim=True)
            w = 1.0 / torch.clamp(d2, min=1e-16)
            yy = (xv[nbr] * w) / w
            return torch.bincount(K * y[q] + yy.argmax(1), minlength=K * K)
        # the reference's CPU path at a 1 M-point subsample: k = 1 search (scipy's cKDTree standing in for
        # torch_cluster, which is not installed) + knn_interpolate's arithmetic + argmax + bincount on the host
        sub = 1_000_000
        p_cpu, v_cpu, c_cpu, y_cpu = pos[:sub].cpu(), v[:sub].cpu(), cnt[:sub].cpu(), y[:sub].cpu()

        def cpu_path():
            from scipy.spatial import cKDTree
            has = c_cpu > 0
            qq = ~has if mode == "own_votes" else torch.ones_like(has)
            _, idx = cKDTree(p_cpu[has].numpy()).query(p_cpu[qq].numpy(), k=1)
            idx = torch.from_numpy(idx)
            diff = p_cpu[has][idx] - p_cpu[qq]
            d2 = (diff * diff).sum(-1, keepdim=True)
            w = 1.0 / torch.clamp(d2, min=1e-16)
            yy = (v_cpu[has][idx] * w) / w
            return np.bincount(K * y_cpu[qq].numpy() + yy.argmax(1).numpy(), minlength=K * K)
        emit(case=f"full_res_{name}", N=NN, cpu_subsample=sub, cpu_path_subsample_ms=host_ms(cpu_path, reps=2), voted=int(voted.numel()), K=K, mode=mode, ms=ours, knn_query_ms=knn,
             fused_kernel_ms=fused, torch_chain_after_knn_ms=gpu_ms(chain, reps=5, warm=1),
             fused_hbm_share=NN * (8 + 4 + K * 4 + 8 + 8) / (fused * 1e-3) / HBM)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
