"""One train step (forward + backward, every parameter's gradient) of ADE20KResNet18TruncatedLayer4 at 1024x512 with
its BatchNorms converted by nn.SyncBatchNorm.convert_sync_batchnorm, against the unconverted encoder:
  * in a 1-rank NCCL group, with the split (all-reduce) path forced (ops.sync_batchnorm_split_at_one_rank): the cost
    of splitting each BatchNorm around its collective, alternated with the fused path in the same process;
  * with two or more GPUs, two NCCL ranks, converted against unconverted (the step time is the slower rank's).
Also the collectives per step and their bytes, computed from the shapes: one all-reduce of 2 C + 1 doubles per
BatchNorm and direction.  Writes profiles/h100_sync_bn.jsonl (or --out) with the card's name and power limit read in
the same run; what could not run here is written with "measured": false.

    python tools/bench_sync_bn.py [--images 2 8] [--reps 5] [--out profiles/h100_sync_bn.jsonl]"""
import argparse
import json
import os
import socket
import subprocess
import sys
import time

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deepviewagg_b200 import ops  # noqa: E402
from deepviewagg_b200.modules.multimodal.modalities import image as I  # noqa: E402

H, W = 512, 1024
MODEL = "ADE20KResNet18TruncatedLayer4"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def collectives(m):
    """(all-reduces per train step, bytes they carry) of the converted m: 2 C + 1 fp64 per BatchNorm and direction."""
    bns = [b for b in m.modules() if isinstance(b, nn.modules.batchnorm._BatchNorm)]
    return 2 * len(bns), sum(2 * 8 * (2 * b.num_features + 1) for b in bns)


def _step(m, x, gy):
    params = [p for p in m.parameters() if p.requires_grad]
    return lambda: torch.autograd.grad(m(x), params, gy)


def _init(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _one_rank(port, images, reps, base, q):
    _init(0, 1, port)
    rows = []
    for B in images:
        torch.manual_seed(0)
        plain = getattr(I, MODEL)().cuda().train()
        synced = nn.SyncBatchNorm.convert_sync_batchnorm(getattr(I, MODEL)().cuda().train())
        synced.load_state_dict(plain.state_dict(), strict=False)
        x = torch.randn(B, 3, H, W, device="cuda")
        with torch.no_grad():
            gy = torch.randn_like(plain(x))
        n, nbytes = collectives(synced)
        res = {"unconverted": [], "split_1rank_nccl": []}
        for _ in range(3):       # alternate the variants
            res["unconverted"].append(timed(_step(plain, x, gy), reps))
            with ops.sync_batchnorm_split_at_one_rank():
                res["split_1rank_nccl"].append(timed(_step(synced, x, gy), reps))
        for k, ts in res.items():
            ms = min(ts)
            rows.append(dict(base, B=B, variant=k, measured=True, ms=ms, ms_per_image=ms / B,
                             collectives_per_step=n if k != "unconverted" else 0,
                             collective_bytes_per_step=nbytes if k != "unconverted" else 0))
        del x, gy
        torch.cuda.empty_cache()
    q.put(rows)
    dist.destroy_process_group()


def _two_ranks(rank, world, port, images, reps, base, q):
    _init(rank, world, port)
    rows = []
    for B in images:
        torch.manual_seed(0)
        plain = getattr(I, MODEL)().cuda().train()
        synced = nn.SyncBatchNorm.convert_sync_batchnorm(getattr(I, MODEL)().cuda().train())
        synced.load_state_dict(plain.state_dict(), strict=False)
        x = torch.randn(B, 3, H, W, device="cuda")
        with torch.no_grad():
            gy = torch.randn_like(plain(x))
        n, nbytes = collectives(synced)
        res = {"unconverted_2rank_nccl": [], "converted_2rank_nccl": []}
        for _ in range(3):
            for k, m in (("unconverted_2rank_nccl", plain), ("converted_2rank_nccl", synced)):
                dist.barrier()
                t = torch.tensor([timed(_step(m, x, gy), reps)], device="cuda")
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                res[k].append(float(t))
        for k, ts in res.items():
            ms = min(ts)
            rows.append(dict(base, B=B, images_per_rank=B, variant=k, measured=True, ms=ms, ms_per_image=ms / B,
                             collectives_per_step=n if k.startswith("converted") else 0,
                             collective_bytes_per_step=nbytes if k.startswith("converted") else 0))
    if rank == 0:
        q.put(rows)
    dist.barrier()
    dist.destroy_process_group()


def _spawn(target, nprocs, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=target, args=(*((r, nprocs) if nprocs > 1 else ()), *args, q)) for r in range(nprocs)]
    for p in procs:
        p.start()
    rows = q.get(timeout=3600)
    for p in procs:
        p.join(timeout=300)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, nargs="+", default=[2, 8])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_sync_bn.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
    base = {"model": MODEL, "H": H, "W": W, "gpu": q, "time": time.strftime("%Y-%m-%d")}
    rows = _spawn(_one_rank, 1, _free_port(), args.images, args.reps, base)
    if torch.cuda.device_count() >= 2:
        rows += _spawn(_two_ranks, 2, _free_port(), args.images, args.reps, base)
    else:
        rows.append(dict(base, variant="converted_2rank_nccl", measured=False,
                         reason=f"{torch.cuda.device_count()} GPU visible; two NCCL ranks need two"))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            print(json.dumps(r), flush=True)
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
