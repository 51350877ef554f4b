"""Forward + backward (train-mode BatchNorm, every parameter's gradient, no input gradient) of ADE20KResNet18PPM per
image on libdva_resnet.so and the gather pool of libdva_b200.so, against the reference's arithmetic on cuDNN
(F.conv2d + F.batch_norm + F.max_pool2d + F.adaptive_avg_pool2d + F.interpolate: oracle/image_ppm_oracle.py) with
TF32 allowed and disabled, NCHW and channels-last, alternated in the same process, at the S3DIS 1024x512 and
KITTI-360 1408x376 image sizes with 8 and 32 images.  Two models: "head", the PPM head alone on a fixed conv5 (its
parameters' gradients only), and "encoder", the whole module.  Writes profiles/h100_image_ppm.jsonl (or --out) with
the card's name and power limit read in the same run: time per image, TFLOP/s from the shapes (2 * output pixels *
C_out * k^2 * C_in per convolution pass; three passes per convolution of the head, the trunk's as
tools/bench_image_resnet18.py counts them) and the peak memory allocated by each variant's step.
A last row times the scale-1 branch's resize backward alone (dva_resnet_resize_bwd from h x w to 1 x 1, 512
channels), which sums a whole map per (image, channel) in one thread.

    python tools/bench_image_ppm.py [--reps 2] [--out profiles/h100_image_ppm.jsonl]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deepviewagg_b200 import _lib, ops  # noqa: E402
from deepviewagg_b200.modules.multimodal.modalities import image as I  # noqa: E402
from oracle import image_ppm_oracle as O  # noqa: E402
from tools.bench_image_resnet18 import SHAPES, flops as trunk_flops, timed  # noqa: E402


def head_flops(B, h, w):
    """conv_last and the four 1x1 branch convolutions on s x s maps, three passes each."""
    fl = 3 * 2 * B * h * w * 512 * 9 * 2560
    fl += sum(3 * 2 * B * s * s * 512 * 512 for s in O.SCALES)
    return fl


class _Trunk:
    """The encoder's trunk walk in the shape bench_image_resnet18.flops reads (.conv)."""

    def __init__(self, enc):
        stem = torch.nn.Sequential(enc.conv1, enc.bn1, enc.relu1, enc.conv2, enc.bn2, enc.relu2, enc.conv3, enc.bn3,
                                   enc.relu3, enc.maxpool)
        self.conv = [stem, enc.layer1, enc.layer2, enc.layer3, enc.layer4]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_image_ppm.jsonl"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    rows = []

    def emit(row):
        rows.append(row)
        print(json.dumps(row), flush=True)

    torch.manual_seed(0)
    net = I.ADE20KResNet18PPM().cuda().train()
    sd = {k: (v.detach().requires_grad_(True) if v.is_floating_point() and "running" not in k and "_iter" not in k
              else v.detach().clone()) for k, v in net.state_dict().items()}
    for model in ("head", "encoder"):
        params = list(net.decoder.parameters()) if model == "head" else list(net.parameters())
        leaves = [sd[k] for k, _ in net.named_parameters() if model == "encoder" or k.startswith("decoder.")]
        for label, B, H, W in SHAPES:
            base = {"model": model, "shape": label, "B": B, "H": H, "W": W, "gpu": q, "time": time.strftime("%Y-%m-%d")}
            h, w = [ops.rn_out(ops.rn_out(ops.rn_out(n, 2), 2), 2) for n in (H, W)]
            if model == "head":
                x = torch.relu(torch.randn(B, 512, h, w, device="cuda")).contiguous(memory_format=torch.channels_last)
                ours_fwd = lambda: net.decoder([x])                                       # noqa: E731
                ref_fwd = lambda xx: O.head(xx, sd, True)                                 # noqa: E731
            else:
                x = torch.randn(B, 3, H, W, device="cuda")
                ours_fwd = lambda: net(x)                                                 # noqa: E731
                ref_fwd = lambda xx: O.forward(xx, sd, True)                              # noqa: E731
            gy = torch.randn(B, 512, h, w, device="cuda")

            def ours():
                torch.autograd.grad(ours_fwd(), params, gy)

            def cudnn(cl):
                def f():
                    xx = x.contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format)
                    torch.autograd.grad(ref_fwd(xx), leaves, gy)
                return f
            variants = {"ours": (ours, None)}
            for tf32 in (True, False):
                for cl in (False, True):
                    variants[f"cudnn_tf32{int(tf32)}_{'cl' if cl else 'nchw'}"] = (cudnn(cl), tf32)
            res, peak = {k: [] for k in variants}, {}
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
            fl = head_flops(B, h, w) + (trunk_flops(_Trunk(net.encoder), B, H, W) if model == "encoder" else 0)
            for k, ts in res.items():
                ms = min(ts)
                emit(dict(base, variant=k, ms=ms, ms_per_image=ms / B, tflops=fl / ms / 1e9,
                          gflop_per_image=fl / B / 1e9, peak_gib=peak[k]))
            del x, gy
            torch.cuda.empty_cache()

    # the scale-1 branch's resize backward alone: one thread per (image, channel) sums the h x w gradient slice
    for label, B, H, W in SHAPES:
        h, w = [ops.rn_out(ops.rn_out(ops.rn_out(n, 2), 2), 2) for n in (H, W)]
        dcat = torch.randn(B, h, w, 2560, device="cuda")
        dx = torch.empty(B, 1, 1, 512, device="cuda")
        sh, sw = ops.resize_scale(1, h), ops.resize_scale(1, w)

        def bwd():
            for _ in range(10):
                _lib.launch("dva_resnet_resize_bwd", dcat.device, dcat, 2560, 512, B, 1, 1, 512, h, w, sh, sw, dx)
        ms = timed(bwd, args.reps) / 10
        emit({"model": "resize_bwd_s1", "shape": label, "B": B, "H": H, "W": W, "gpu": q,
              "time": time.strftime("%Y-%m-%d"), "variant": "ours", "ms": ms, "ms_per_image": ms / B,
              "gbps_read": B * h * w * 512 * 4 / ms / 1e6})
        del dcat
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
