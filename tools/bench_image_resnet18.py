"""Forward + backward (train-mode BatchNorm, every parameter's gradient, no input gradient) of the ADE20K ResNet-18
encoders per image, ADE20KResNet18TruncatedLayer4 and ADE20KResNet18Pyramid(scale_factor=1) on libdva_resnet.so,
against the reference's arithmetic on cuDNN (F.conv2d + F.batch_norm + F.max_pool2d + F.interpolate:
oracle/image_resnet18_oracle.py) with TF32 allowed and disabled, NCHW and channels-last, alternated in the same
process, at the S3DIS 1024x512 and KITTI-360 1408x376 image sizes with 8 and 32 images.  Writes
profiles/h100_image_resnet18.jsonl (or --out) with the card's name and power limit read in the same run: time per
image, and FLOP/s computed from the shapes (2 * output pixels * C_out * k^2 * C_in per convolution pass; three passes
per convolution, two for the stem's first, whose input needs no gradient).

    python tools/bench_image_resnet18.py [--reps 2] [--out profiles/h100_image_resnet18.jsonl]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deepviewagg_b200 import ops  # noqa: E402
from deepviewagg_b200.modules.multimodal.modalities import image as I  # noqa: E402
from oracle import image_resnet18_oracle as O  # noqa: E402

SHAPES = [("s3dis_1024x512", 8, 512, 1024), ("s3dis_1024x512", 32, 512, 1024),
          ("kitti360_1408x376", 8, 376, 1408), ("kitti360_1408x376", 32, 376, 1408)]
MODELS = [("TruncatedLayer4", lambda: I.ADE20KResNet18TruncatedLayer4()),
          ("Pyramid_sf1", lambda: I.ADE20KResNet18Pyramid(scale_factor=1))]


def flops(net, B, H, W):
    """Forward + both backward passes of every convolution, from the shapes (the stem's first has no dgrad)."""
    fl = 0

    def conv(c, Ho, Wo, passes=3):
        nonlocal fl
        fl += passes * 2 * B * Ho * Wo * c.out_channels * c.kernel_size[0] ** 2 * c.in_channels

    for layer in net.conv:
        if isinstance(layer[0], I.BasicBlock):
            for blk in layer:
                H, W = ops.rn_out(H, blk.conv1.stride[0]), ops.rn_out(W, blk.conv1.stride[0])
                for c in [blk.conv1, blk.conv2] + ([blk.downsample[0]] if blk.downsample is not None else []):
                    conv(c, H, W)
        else:
            for i in (0, 3, 6):
                H, W = ops.rn_out(H, layer[i].stride[0]), ops.rn_out(W, layer[i].stride[0])
                conv(layer[i], H, W, 2 if i == 0 and layer is net.conv[0] else 3)
            H, W = ops.rn_out(H, 2), ops.rn_out(W, 2)
    return fl


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
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_image_resnet18.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    rows = []
    for mname, build in MODELS:
        torch.manual_seed(0)
        net = build().cuda().train()
        params = list(net.parameters())
        sd = {k: (v.detach().requires_grad_(True) if v.is_floating_point() and "running" not in k and "_iter" not in k
                  else v.detach().clone()) for k, v in net.state_dict().items()}
        leaves = [sd[k] for k, _ in net.named_parameters()]
        pyramid = isinstance(net, I.ADE20KResNet18Pyramid)
        for label, B, H, W in SHAPES:
            base = {"model": mname, "shape": label, "B": B, "H": H, "W": W, "gpu": q, "time": time.strftime("%Y-%m-%d")}
            x = torch.randn(B, 3, H, W, device="cuda")
            with torch.no_grad():
                gy = torch.randn_like(net(x))

            def ours():
                torch.autograd.grad(net(x), params, gy)

            def cudnn(cl):
                def f():
                    xx = x.contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format)
                    y = O.forward(xx, sd, net._LAYERS, True, net.scale_factor, pyramid)
                    torch.autograd.grad(y, leaves, gy)
                return f
            variants = {"ours": (ours, None)}
            for tf32 in (True, False):
                for cl in (False, True):
                    variants[f"cudnn_tf32{int(tf32)}_{'cl' if cl else 'nchw'}"] = (cudnn(cl), tf32)
            res = {k: [] for k in variants}
            for _ in range(2):     # alternate the variants
                for k, (fn, tf32) in variants.items():
                    if tf32 is not None:
                        torch.backends.cudnn.allow_tf32 = tf32
                    try:
                        res[k].append(timed(fn, args.reps))
                    except torch.OutOfMemoryError:
                        res[k].append(float("nan"))
                    torch.backends.cudnn.allow_tf32 = True
                    torch.cuda.empty_cache()
            fl = flops(net, B, H, W)
            for k, ts in res.items():
                ms = min(ts)
                row = dict(base, variant=k, ms=ms, ms_per_image=ms / B, tflops=fl / ms / 1e9,
                           gflop_per_image=fl / B / 1e9)
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
