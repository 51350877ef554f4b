"""No3D hot paths on the H100: the query / search k-NN (mapping.knn_query, nearest seen point of every
unseen point) and the CSR log-softmax NLL (ops.csr_nll_loss), each against what a user would write in
torch on the same GPU.

    python tools/bench_no3d.py --out profiles/h100_no3d.jsonl

k-NN workloads (k = 1): a room-like cloud (floor, ceiling and four walls of a 10 x 8 x 3 m room) and a
street-cylinder-like cloud (road and two facades in a 20 m radius cylinder), with 100 k and 1 M search
points.  The seen set covers only part of the scene (one camera's half of the room / one side of the street
and a stretch of road); the queries are unseen points, about half as many as the search points, so most
are metres away from every seen point.  The comparison is a chunked dense torch.cdist + argmin.  Both are
timed with CUDA events over --reps calls after a warm-up; the k-NN rows also check that every returned
distance is exact and at most the one cdist's choice has.

NLL workload: the S3DIS step shape (1.15 M views x 13 classes, fp32, ~3 views per point, 10 % ignored
labels): forward + backward of ops.csr_nll_loss against repeat_interleave + log_softmax + nll_loss and its
backward, with the loss and gradient compared.  Algorithmic bytes: forward V K 4 (logits) + V 4 (lse) + 16 N
(labels, pointers); backward 2 V K 4 + V 4 + 16 N; the HBM share is their time at 3.35 TB/s over the
measured time.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepviewagg_b200 import ops  # noqa: E402
from deepviewagg_b200.core.multimodal.mapping import knn_query  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("unknown", "unknown")
    return name, power


def timed(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, out


def room(n, gen):
    """floor, ceiling and four walls of a 10 x 8 x 3 m room; seen: the half x < 4 (one camera)."""
    L = torch.tensor([10.0, 8.0, 3.0])
    face = torch.randint(0, 6, (n,), generator=gen)
    p = torch.rand(n, 3, generator=gen) * L
    axis = face // 2
    p[torch.arange(n), axis] = torch.where(face % 2 == 0, 0.0, L[axis])
    seen = p[:, 0] < 4.0
    return p, seen


def street(n, gen):
    """road (z = 0, |y| < 6) and two facades (|y| = 6, z < 15) along x in [-20, 20]; seen: the facade
    y = +6 and the road ahead of the sensor (x in [-8, 8], y > 0)."""
    u = torch.rand(n, 3, generator=gen)
    kind = torch.randint(0, 3, (n,), generator=gen)
    x = u[:, 0] * 40 - 20
    p = torch.stack([x, u[:, 1] * 12 - 6, torch.zeros(n)], 1)
    fac = kind > 0
    p[fac, 1] = torch.where(kind[fac] == 1, 6.0, -6.0)
    p[fac, 2] = u[fac, 2] * 15
    seen = ((p[:, 1] == 6.0) & fac) | ((~fac) & (p[:, 0].abs() < 8) & (p[:, 1] > 0))
    return p, seen


def cdist_argmin(q, s, chunk):
    out = torch.empty(q.shape[0], dtype=torch.int64, device=q.device)
    for i in range(0, q.shape[0], chunk):
        out[i:i + chunk] = torch.cdist(q[i:i + chunk], s).argmin(dim=1)
    return out


def exact_d2(q, s):
    d = q - s
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def bench_knn(name, maker, n_search, reps, gen):
    n_total = int(n_search * 1.6)
    while True:
        p, seen = maker(n_total, gen)
        if int(seen.sum()) >= n_search and int((~seen).sum()) >= n_search // 2:
            break
        n_total = int(n_total * 1.3)
    s = p[seen][:n_search].cuda()
    q = p[~seen][:n_search // 2].cuda()
    t_knn, nbr = timed(lambda: knn_query(q, s, 1), reps)
    chunk = max(1, int(2 ** 31 // (4 * s.shape[0])))
    t_cd, idx = timed(lambda: cdist_argmin(q, s, chunk), 1, warmup=1)
    d_ours, d_cd = exact_d2(q, s[nbr[:, 0]]), exact_d2(q, s[idx])
    far = exact_d2(q, s[nbr[:, 0]]).sqrt()
    return dict(workload=f"knn_query_{name}_{n_search // 1000}k", k=1, n_search=int(s.shape[0]),
                n_query=int(q.shape[0]), ms=round(t_knn, 3), cdist_argmin_ms=round(t_cd, 2),
                speedup=round(t_cd / t_knn, 1), median_nn_dist_m=round(float(far.median()), 3),
                not_farther_than_cdist=bool((d_ours <= d_cd).all()),
                same_index_share=round(float((nbr[:, 0] == idx).float().mean()), 6))


def bench_nll(reps, gen):
    V_target, K = 1_150_000, 13
    n = V_target // 3
    counts = torch.poisson(torch.full((n,), 3.0), generator=gen).long()
    csr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)]).cuda()
    V = int(csr[-1])
    logits = (3 * torch.randn(V, K, generator=gen)).cuda()
    labels = torch.randint(0, K, (n,), generator=gen)
    labels[torch.rand(n, generator=gen) < 0.1] = -1
    labels = labels.cuda()

    def ours():
        x = logits.detach().requires_grad_(True)
        loss = ops.csr_nll_loss(x, labels, csr)
        g, = torch.autograd.grad(loss, x)
        return loss, g

    def chain():
        x = logits.detach().requires_grad_(True)
        target = torch.repeat_interleave(labels, csr[1:] - csr[:-1])
        loss = torch.nn.functional.nll_loss(torch.log_softmax(x, -1), target, ignore_index=-1)
        g, = torch.autograd.grad(loss, x)
        return loss, g

    t_ours, (l1, g1) = timed(ours, reps)
    t_chain, (l2, g2) = timed(chain, reps)
    x64 = logits.double().requires_grad_(True)
    l64 = torch.nn.functional.nll_loss(torch.log_softmax(x64, -1),
                                       torch.repeat_interleave(labels, csr[1:] - csr[:-1]), ignore_index=-1)
    g64, = torch.autograd.grad(l64, x64)
    byts = V * K * 4 + V * 4 + 16 * n + 2 * V * K * 4 + V * 4 + 16 * n
    return dict(workload="csr_nll_loss_s3dis_step", V=V, N=n, K=K, ms_fwd_bwd=round(t_ours, 4),
                torch_chain_ms=round(t_chain, 4), speedup=round(t_chain / t_ours, 2),
                hbm_share=round(byts / HBM_BYTES_PER_S / (t_ours * 1e-3), 3),
                loss_rel_err_vs_fp64=float(abs(float(l1.detach()) - float(l64)) / abs(float(l64))),
                torch_chain_loss_rel_err_vs_fp64=float(abs(float(l2.detach()) - float(l64)) / abs(float(l64))),
                grad_max_err_vs_fp64=float((g1.double() - g64).abs().max()),
                torch_chain_grad_max_err_vs_fp64=float((g2.double() - g64).abs().max()),
                bit_identical_rerun=bool(torch.equal(ours()[1], g1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_no3d.jsonl")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="100000,1000000")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_no3d measures on the GPU; no CUDA device found")
    name, power = card()
    gen = torch.Generator().manual_seed(0)
    rows = []
    for n_search in [int(v) for v in args.sizes.split(",")]:
        for wname, maker in (("room", room), ("street", street)):
            rows.append(bench_knn(wname, maker, n_search, args.reps, gen))
            print(json.dumps(rows[-1]), flush=True)
    rows.append(bench_nll(max(20, args.reps), gen))
    print(json.dumps(rows[-1]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            r.update(gpu=name, power_limit=power, torch=torch.__version__)
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
