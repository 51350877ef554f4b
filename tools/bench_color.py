"""Colour transforms on the H100: ColorJitter, ToFloatImage and Normalize on CUDA (dva_color_jitter_u8,
dva_image_to_float) against the package's torch restatement run on CUDA tensors (the multi-pass chain a user
would write) and against the CPU path on all host threads.

    python tools/bench_color.py --out profiles/h100_color.jsonl

Workloads, channels-last uint8 as LoadImages produces them:
  s3dis       4 x 1024 x 512   (an S3DIS sample)
  kitti360    16 x 704 x 188   (a KITTI-360 sample at its configured resolution and image count)
  bandwidth   64 x 1024 x 512  (large enough for the HBM bound)
The jitter runs the S3DIS factors with contrast in the middle of the order (both passes).  Times are CUDA events
over `--reps` calls after a warm-up (op calls: the output allocation is included), and a host clock for the CPU
path.  Algorithmic bytes: jitter 3 B H W (sum pass, contrast only) + 6 B H W (apply pass); ToFloatImage 15 B per
pixel; Normalize 24 B per pixel; the HBM share is their time at 3.35 TB/s over the measured time.  Every row also
checks the CUDA result against the torch restatement bit for bit.  The card name and power limit are read in the
same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepviewagg_b200 import ops  # noqa: E402
from deepviewagg_b200.core.multimodal.transforms import color_jitter_torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
WORKLOADS = {"s3dis": (4, 512, 1024), "kitti360": (16, 188, 704), "bandwidth": (64, 512, 1024)}
JITTER = [("saturation", 1.37), ("contrast", 0.62), ("brightness", 1.21)]
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("unknown", "unknown")
    return name, power


def time_events(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def time_host(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) * 1e3 / reps


def algorithmic_bytes(op, B, H, W):
    px = B * H * W
    if op == "color_jitter":
        return (3 if any(n == "contrast" for n, _ in JITTER) else 0) * px + 6 * px
    return {"to_float": 15, "normalize": 24}[op] * px


def run(tag, B, H, W, reps, cpu_reps):
    g = torch.Generator().manual_seed(0)
    x_cpu = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g).contiguous(
        memory_format=torch.channels_last)
    x = x_cpu.cuda()
    f = ops.image_to_float(x)
    mean_d, std_d = torch.tensor(MEAN, device="cuda").view(-1, 1, 1), torch.tensor(STD, device="cuda").view(-1, 1, 1)
    mean_h, std_h = torch.tensor(MEAN).view(-1, 1, 1), torch.tensor(STD).view(-1, 1, 1)
    f_cpu = x_cpu.float() / 255
    cases = {
        "color_jitter": (lambda: ops.color_jitter_u8(x, JITTER), lambda: color_jitter_torch(x, JITTER),
                         lambda: color_jitter_torch(x_cpu, JITTER)),
        "to_float": (lambda: ops.image_to_float(x), lambda: x.float() / torch.full((), 255.0, device="cuda"),
                     lambda: x_cpu.float() / 255),
        "normalize": (lambda: ops.image_to_float(f, MEAN, STD), lambda: (f - mean_d) / std_d,
                      lambda: (f_cpu - mean_h) / std_h),
    }
    rows = []
    for op, (kern, torch_cuda, cpu) in cases.items():
        exact = bool(torch.equal(kern(), torch_cuda()))
        t_k = time_events(kern, reps)
        t_t = time_events(torch_cuda, reps)
        t_c = time_host(cpu, cpu_reps)
        nbytes = algorithmic_bytes(op, B, H, W)
        rows.append(dict(workload=tag, op=op, images=B, size=[W, H], layout="channels_last", kernel_ms=round(t_k, 4),
                         torch_cuda_ms=round(t_t, 4), cpu_ms=round(t_c, 2), cpu_threads=torch.get_num_threads(),
                         algorithmic_bytes=nbytes, achieved_tb_s=round(nbytes / (t_k * 1e-3) / 1e12, 3),
                         hbm_share=round(nbytes / HBM_BYTES_PER_S / (t_k * 1e-3), 3), equal_to_torch=exact))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_color.jsonl")
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--cpu-reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_color.py measures the CUDA kernels: no CUDA device")
    name, power = card()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fo:
        for tag, (B, H, W) in WORKLOADS.items():
            for r in run(tag, B, H, W, args.reps, args.cpu_reps):
                r.update(gpu=name, power_limit=power, torch=torch.__version__)
                fo.write(json.dumps(r) + "\n")
                print(json.dumps(r))


if __name__ == "__main__":
    main()
