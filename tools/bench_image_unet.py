"""Forward + backward of the full shipped image UNet (in_feat = 32, 5 down / 5 up stages as Res16UNet21-15_light,
last_conv 1x1 to 13 classes) in fp32, UNet on libdva_conv2d.so + libdva_unet.so against the same layers on cuDNN
(F.pad reflect + F.conv2d, F.conv_transpose2d, F.group_norm: the reference's arithmetic, oracle/image_unet_oracle.py)
with TF32 allowed and disabled, NCHW and channels-last, alternated in the same process.  Writes
profiles/h100_image_unet.jsonl (or --out): time per image, and FLOP/s and bytes/s computed from the shapes (FLOPs
2 * pixels * C_out * R * S * C_in per convolution pass, counted on the input pixels for the 2x2 upsampling, three
passes per convolution; bytes: each pass reads its input map and writes its output map once, fp32).

    python tools/bench_image_unet.py [--reps 3] [--out profiles/h100_image_unet.jsonl]"""
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

from deepviewagg_b200.modules.multimodal.modalities.image import UNet  # noqa: E402
from oracle import image_unet_oracle as O  # noqa: E402
from test_image_unet_oracle import DOWN, UP, small_opt  # noqa: E402

# (label, B, H, W): S3DIS 1024 x 512 images, 8 and 32 of them; KITTI-360 1408 x 376 (376 is not a multiple of 16:
# the UNet raises, and the timing uses the 1408 x 368 crop); many 64 x 64 crops
SHAPES = [("s3dis_1024x512", 8, 512, 1024), ("s3dis_1024x512", 32, 512, 1024),
          ("kitti360_1408x376", 8, 376, 1408), ("kitti360_1408x368_crop", 8, 368, 1408),
          ("crops_64x64", 1024, 64, 64)]


def flops_bytes(net, B, H, W):
    fl = by = 0

    def conv(Ci, Co, k, Hi, Wi, Ho, Wo, per_in=False):
        nonlocal fl, by
        pixels = Hi * Wi if per_in else Ho * Wo
        taps = 4 if per_in else k * k
        fl += 3 * 2 * B * pixels * Co * taps * Ci
        by += 3 * 4 * B * (Hi * Wi * Ci + Ho * Wo * Co)

    def blocks(st, H, W, transposed):
        for blk in (st.blocks or []):
            w1, w2 = blk.block[0].weight, blk.block[3].weight
            Ci, Co = (w1.shape[0], w1.shape[1]) if transposed else (w1.shape[1], w1.shape[0])
            conv(Ci, Co, 3, H, W, H, W)
            conv(Co, Co, 3, H, W, H, W)
            if blk.downsample is not None:
                conv(Ci, Co, 1, H, W, H, W)

    for st in net.down_modules:
        w = st.conv_in[0].weight
        k, s = w.shape[-1], st.conv_in[0].stride[0]
        conv(w.shape[1], w.shape[0], k, H, W, H // s, W // s)
        H, W = H // s, W // s
        blocks(st, H, W, False)
    for st in net.up_modules:
        w = st.conv_in[0].weight
        k, s = w.shape[-1], st.conv_in[0].stride[0]
        conv(w.shape[0], w.shape[1], k, H, W, H * s, W * s, per_in=s == 2)
        H, W = H * s, W * s
        blocks(st, H, W, True)
    w = net.last.conv.weight
    conv(w.shape[1], w.shape[0], 1, H, W, H, W)
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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_image_unet.jsonl"))
    ap.add_argument("--shapes", default="all")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    torch.manual_seed(0)
    net = UNet(small_opt("unet5", 32)).cuda()
    params = list(net.parameters())
    sd = {k: v.detach().requires_grad_(True) for k, v in net.state_dict().items()}
    shapes = SHAPES if args.shapes == "all" else [s for s in SHAPES if s[0] in args.shapes.split(",")]
    rows = []
    for label, B, H, W in shapes:
        base = {"shape": label, "B": B, "H": H, "W": W, "gpu": q, "time": time.strftime("%Y-%m-%d")}
        try:
            net.check_sizes(H, W)
        except ValueError as e:
            row = dict(base, variant="ours", error=f"ValueError: {e}")
            rows.append(row)
            print(json.dumps(row), flush=True)
            continue
        x = torch.randn(B, 4, H, W, device="cuda")
        gy = torch.randn(B, 13, H, W, device="cuda")

        def ours():
            xx = x.detach().requires_grad_(True)
            torch.autograd.grad(net(xx), [xx] + params, gy)

        def cudnn(cl):
            def f():
                xx = x.detach().contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format)
                xx.requires_grad_(True)
                y = O.unet(xx, sd, DOWN, UP["unet5"], last={})
                torch.autograd.grad(y, [xx] + list(sd.values()), gy)
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
        fl, by = flops_bytes(net, B, H, W)
        for k, ts in res.items():
            ms = min(ts)
            row = dict(base, variant=k, ms=ms, ms_per_image=ms / B, tflops=fl / ms / 1e9, gbps=by / ms / 1e6,
                       gflop_per_image=fl / B / 1e9)
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
