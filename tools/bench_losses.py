"""Loss of the sparse-conv models on the H100: cross-entropy (ops.csr_nll_loss, with and without class weights)
plus Lovász-softmax (ops.lovasz_softmax on log-probabilities), forward + backward, against the torch chain a
reference training step runs on the same GPU.

    python tools/bench_losses.py --out profiles/h100_losses.jsonl

Workloads: the S3DIS step shape (383 k points x 13 classes, 10 % ignored labels), the same with 20 classes
(ScanNet), and the S3DIS shape with class weights.  Per workload, with logits [P, K] fp32 requiring grad:
  ours   output = log_softmax(logits); csr_nll_loss(logits, y, weight=w) + lovasz_softmax(output, y,
         log_probs=True); backward
  chain  output = log_softmax(logits); F.nll_loss(output, y, weight=w, ignore_index=-1) + the reference's
         lovasz_softmax(output.exp(), y, ignore=-1) (metrics/lovasz_loss.py:155-230, restated below: one sort,
         gather, cumsum and dot per class, on CUDA tensors); backward
Also timed alone: the Lovász forward + backward, the NLL forward + backward, and the stable segmented sort of the
[K, P] key matrix inside the Lovász forward (torch.sort, i.e. CUB's segmented radix sort), whose share of the
Lovász time is reported.  Times are CUDA events over --reps calls after a warm-up; losses and gradients of both
paths are compared.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepviewagg_b200 import ops  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("unknown", "unknown")
    return name, power


def timed(fn, reps, warmup=3):
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


def torch_lovasz(probas, labels, ignore=-1):
    """lovasz_softmax_flat(*flatten_probas(probas, labels, ignore), classes='present') in torch."""
    valid = labels != ignore
    probas, labels = probas[valid], labels[valid]
    losses = []
    for c in range(probas.shape[1]):
        fg = (labels == c).float()
        if fg.sum() == 0:
            continue
        errors = (fg - probas[:, c]).abs()
        errors_sorted, perm = torch.sort(errors, 0, descending=True)
        fg_sorted = fg[perm]
        gts = fg_sorted.sum()
        intersection = gts - fg_sorted.cumsum(0)
        union = gts + (1 - fg_sorted).cumsum(0)
        jaccard = 1.0 - intersection / union
        jaccard[1:] = jaccard[1:] - jaccard[:-1]
        losses.append(torch.dot(errors_sorted, jaccard))
    return sum(losses) / len(losses) if losses else probas.sum() * 0


def bench(name, P, K, weighted, reps, gen):
    logits = (2 * torch.randn(P, K, generator=gen)).cuda()
    y = torch.randint(0, K, (P,), generator=gen)
    y[torch.rand(P, generator=gen) < 0.1] = -1
    y = y.cuda()
    w = (torch.rand(K, generator=gen) + 0.5).cuda() if weighted else None

    def ours():
        x = logits.detach().requires_grad_(True)
        out = F.log_softmax(x, dim=-1)
        loss = ops.csr_nll_loss(x, y, None, -1, weight=w) + ops.lovasz_softmax(out, y, log_probs=True)
        loss.backward()
        return loss.detach(), x.grad

    def chain():
        x = logits.detach().requires_grad_(True)
        out = F.log_softmax(x, dim=-1)
        loss = F.nll_loss(out, y, weight=w, ignore_index=-1) + torch_lovasz(out.exp(), y, ignore=-1)
        loss.backward()
        return loss.detach(), x.grad

    def lovasz_only():
        x = F.log_softmax(logits, dim=-1).detach().requires_grad_(True)
        loss = ops.lovasz_softmax(x, y, log_probs=True)
        loss.backward()
        return loss

    def nll_only():
        x = logits.detach().requires_grad_(True)
        loss = ops.csr_nll_loss(x, y, None, -1, weight=w)
        loss.backward()
        return loss

    keys = torch.rand(K, P, device="cuda")

    def sort_only():
        return torch.sort(keys, dim=1, descending=True, stable=True)

    ms, (l_ours, g_ours) = timed(ours, reps)
    ms_chain, (l_chain, g_chain) = timed(chain, reps)
    ms_lov, _ = timed(lovasz_only, reps)
    ms_nll, _ = timed(nll_only, reps)
    ms_sort, _ = timed(sort_only, reps)
    return dict(workload=name, points=P, classes=K, ignored=0.1, weighted=weighted, ms=round(ms, 4),
                chain_ms=round(ms_chain, 4), speedup=round(ms_chain / ms, 2), lovasz_fwd_bwd_ms=round(ms_lov, 4),
                nll_fwd_bwd_ms=round(ms_nll, 4), sort_ms=round(ms_sort, 4),
                sort_share_of_lovasz=round(ms_sort / ms_lov, 3), sort_share_of_step_loss=round(ms_sort / ms, 3),
                loss_rel_diff=float(abs(l_ours - l_chain) / abs(l_chain)),
                grad_max_abs_diff=float((g_ours - g_chain).abs().max()),
                grad_max_abs=float(g_chain.abs().max()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_losses.jsonl")
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_losses.py measures on a GPU; none is visible")
    name, power = card()
    gen = torch.Generator().manual_seed(0)
    rows = [bench("s3dis_383k_13", 383_000, 13, False, args.reps, gen),
            bench("scannet_383k_20", 383_000, 20, False, args.reps, gen),
            bench("s3dis_383k_13_weighted", 383_000, 13, True, args.reps, gen)]
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            r.update(gpu=name, power_limit=power, torch=torch.__version__)
            f.write(json.dumps(r) + "\n")
            print(json.dumps(r))


if __name__ == "__main__":
    main()
