"""Forward + backward of the five-stage shipped image encoder (in_feat = 32: 4 -> 32 -> 32 -> 64 -> 128 -> 256,
N = [0, 2, 2, 2, 2]) in fp32, ResNetDown on libdva_conv2d.so against the same layers on cuDNN (F.pad reflect +
F.conv2d + F.group_norm, the reference's arithmetic) with TF32 allowed and disabled, NCHW and channels-last,
alternated in the same process.  Writes profiles/h100_image_encoder.jsonl (or --out): time per image, and FLOP/s and
bytes/s computed from the shapes (FLOPs 2 * B * H' * W' * C_out * R * S * C_in per convolution pass, three passes
per convolution; bytes: each pass reads its input map and writes its output map once, fp32).

    python tools/bench_image_encoder.py [--reps 5] [--out profiles/h100_image_encoder.jsonl]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import image_encoder_oracle as O  # noqa: E402
from test_gpu_image_encoder import KERNEL, PADDING, STRIDE, encoder  # noqa: E402

# (label, B, H, W): S3DIS 1024 x 512 and KITTI-360 1408 x 376 images, 8 and 32 of them, and many 64 x 64 crops
SHAPES = [("s3dis_1024x512", 8, 512, 1024), ("s3dis_1024x512", 32, 512, 1024), ("kitti360_1408x376", 8, 376, 1408),
          ("kitti360_1408x376", 32, 376, 1408), ("crops_64x64", 1024, 64, 64)]


def flops_bytes(stages, B, H, W):
    fl = by = 0
    for i, st in enumerate(stages):
        convs = [(st.conv_in[0], KERNEL[i], STRIDE[i])]
        for blk in (st.blocks or []):
            convs += [(blk.block[0], 3, 1), (blk.block[3], 3, 1)]
            if blk.downsample is not None:
                convs.append((blk.downsample[0], 1, 1))
        for conv, k, s in convs:
            Co, Ci = conv.weight.shape[:2]
            Ho, Wo = H // s, W // s
            fl += 3 * 2 * B * Ho * Wo * Co * k * k * Ci
            by += 3 * 4 * B * (H * W * Ci + Ho * Wo * Co)
        H, W = H // STRIDE[i], W // STRIDE[i]
    return fl, by


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_image_encoder.jsonl"))
    ap.add_argument("--shapes", default="all")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    stages = encoder(32)
    sds = [{k: v.detach().requires_grad_(True) for k, v in st.state_dict().items()} for st in stages]
    shapes = SHAPES if args.shapes == "all" else [s for s in SHAPES if s[0] in args.shapes.split(",")]
    rows = []
    for label, B, H, W in shapes:
        x = torch.randn(B, 4, H, W, device="cuda")
        gy = torch.randn(B, 256, H // 16, W // 16, device="cuda")
        params = [p for st in stages for p in st.parameters()]

        def ours():
            xx = x.detach().requires_grad_(True)
            torch.autograd.grad(stages(xx), [xx] + params, gy)

        def cudnn(tf32, cl):
            def f():
                xx = x.detach().contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format)
                xx.requires_grad_(True)
                y = O.encoder(xx, [(sd, KERNEL[i], STRIDE[i], PADDING[i]) for i, sd in enumerate(sds)])
                torch.autograd.grad(y, [xx] + [p for sd in sds for p in sd.values()], gy)
            return f
        variants = {"ours": ours}
        for tf32 in (True, False):
            for cl in (False, True):
                variants[f"cudnn_tf32{int(tf32)}_{'cl' if cl else 'nchw'}"] = (cudnn(tf32, cl), tf32)
        res = {k: [] for k in variants}
        for _ in range(2):     # alternate the variants
            for k, v in variants.items():
                fn, tf32 = (v, None) if k == "ours" else v
                if tf32 is not None:
                    torch.backends.cudnn.allow_tf32 = tf32
                try:
                    res[k].append(timed(fn, args.reps))
                except torch.OutOfMemoryError:
                    res[k].append(float("nan"))
                torch.backends.cudnn.allow_tf32 = True
                torch.cuda.empty_cache()
        fl, by = flops_bytes(stages, B, H, W)
        for k, ts in res.items():
            ms = min(ts)
            row = {"shape": label, "B": B, "H": H, "W": W, "variant": k, "ms": ms, "ms_per_image": ms / B,
                   "tflops": fl / ms / 1e9, "gbps": by / ms / 1e6, "gpu": q, "time": time.strftime("%Y-%m-%d")}
            rows.append(row)
            print(json.dumps(row), flush=True)
        del x, gy
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
