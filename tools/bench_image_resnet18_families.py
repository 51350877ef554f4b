"""Forward + backward (train-mode BatchNorm, every parameter's gradient, no input gradient) of the ImageNet and
Cityscapes ResNet-18 encoders per image on libdva_resnet.so -- ResNet18TruncatedLayer0 (the image encoder of the
shipped sparse-conv fusion configs), ResNet18TruncatedLayer4, CityscapesResNet18TruncatedLayer4 and the
[CityscapesResNet18Layer0, ..., Layer4] chain of the multi-scale configs -- against the reference's arithmetic on
cuDNN (F.conv2d + F.batch_norm + F.max_pool2d: oracle/image_resnet18_families_oracle.py) with TF32 allowed and
disabled, NCHW and channels-last, alternated in the same process, at 1024x512 and 1408x376 with 8 and 32 images.
For ResNet18TruncatedLayer0 a torch.profiler run splits the step's kernel time by kernel.  Writes
profiles/h100_image_resnet18_families.jsonl (or --out) with the card's name and power limit read in the same run.

    python tools/bench_image_resnet18_families.py [--reps 2] [--out profiles/h100_image_resnet18_families.jsonl]"""
import argparse
import collections
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deepviewagg_b200.modules.multimodal.modalities import image as I  # noqa: E402
from oracle import image_resnet18_families_oracle as O  # noqa: E402

SHAPES = [("s3dis_1024x512", 8, 512, 1024), ("s3dis_1024x512", 32, 512, 1024),
          ("kitti360_1408x376", 8, 376, 1408), ("kitti360_1408x376", 32, 376, 1408)]
MODELS = [("ResNet18TruncatedLayer0", lambda: [I.ResNet18TruncatedLayer0()]),
          ("ResNet18TruncatedLayer4", lambda: [I.ResNet18TruncatedLayer4()]),
          ("CityscapesResNet18TruncatedLayer4", lambda: [I.CityscapesResNet18TruncatedLayer4()]),
          ("CityscapesResNet18Layer0-4", lambda: [getattr(I, f"CityscapesResNet18Layer{i}")() for i in range(5)])]


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


def kernel_split(fn):
    """{kernel name: total CUDA ms} of one fn() under torch.profiler."""
    fn()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        fn()
        torch.cuda.synchronize()
    out = collections.defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            out[e.name] += e.device_time_total / 1e3
    return dict(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_image_resnet18_families.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    rows = []
    for mname, build in MODELS:
        torch.manual_seed(0)
        nets = [n.cuda().train() for n in build()]
        params = [p for n in nets for p in n.parameters()]
        sds = [{k: (v.detach().requires_grad_(True) if v.is_floating_point() and "running" not in k
                    else v.detach().clone()) for k, v in n.state_dict().items()} for n in nets]
        leaves = [sd[k] for n, sd in zip(nets, sds) for k, _ in n.named_parameters()]
        fam = "cityscapes" if mname.startswith("Cityscapes") else "imagenet"

        def ours_fwd(x):
            for n in nets:
                x = n(x)
            return x

        for label, B, H, W in SHAPES:
            base = {"model": mname, "shape": label, "B": B, "H": H, "W": W, "gpu": q, "time": time.strftime("%Y-%m-%d")}
            x = torch.randn(B, 3, H, W, device="cuda")
            with torch.no_grad():
                gy = torch.randn_like(ours_fwd(x))

            def ours():
                torch.autograd.grad(ours_fwd(x), params, gy)

            def cudnn(cl):
                def f():
                    y = x.contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format)
                    for n, sd in zip(nets, sds):
                        y = O.forward(y, sd, fam, n._LAYERS, True, momentum=0.1)
                    torch.autograd.grad(y, leaves, gy)
                return f
            variants = {"ours": (ours, None)}
            for tf32 in (True, False):
                for cl in (False, True):
                    variants[f"cudnn_tf32{int(tf32)}_{'cl' if cl else 'nchw'}"] = (cudnn(cl), tf32)
            res = {k: [] for k in variants}
            peak = {}
            for _ in range(2):     # alternate the variants
                for k, (fn, tf32) in variants.items():
                    if tf32 is not None:
                        torch.backends.cudnn.allow_tf32 = tf32
                    torch.cuda.reset_peak_memory_stats()
                    try:
                        res[k].append(timed(fn, args.reps))
                    except torch.OutOfMemoryError:
                        res[k].append(float("nan"))
                    peak[k] = torch.cuda.max_memory_allocated() / 2 ** 30
                    torch.backends.cudnn.allow_tf32 = True
                    torch.cuda.empty_cache()
            for k, ts in res.items():
                ms = min(ts)
                row = dict(base, variant=k, ms=ms, ms_per_image=ms / B, peak_gib=peak[k])
                rows.append(row)
                print(json.dumps(row), flush=True)
            if mname == "ResNet18TruncatedLayer0":
                split = kernel_split(ours)
                total = sum(split.values())
                row = dict(base, variant="ours_kernel_split", kernel_ms_total=total,
                           kernels={k: round(v, 4) for k, v in sorted(split.items(), key=lambda kv: -kv[1])})
                rows.append(row)
                print(json.dumps(row), flush=True)
            del x, gy
            torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
