"""Image loading on the H100: host decode, H2D copy and kernel time of the CUDA read_images path
(dva_resample_u8, dva_nonstatic_mask) against Pillow's resize on the host's threads.

    python tools/bench_images.py --out profiles/h100_images.jsonl

Workloads (synthetic PNGs written to a temporary directory, smooth fields plus noise):
  s3dis_load   8 panoramas 4096 x 2048 -> 1024 x 512   (LoadImages at the S3DIS ref_size)
  s3dis_mask   5 panoramas 4096 x 2048 -> 2048 x 1024  (NonStaticMask at proj_upscale 2) + the mask kernel
  kitti_load   16 images 1408 x 376 -> 704 x 188
Kernel times are CUDA events over `--reps` launches after a warm-up.  The HBM share is the algorithmic bytes
(input rows read + 2 x the uint8 temporary + output) over kernel time, against 3.35 TB/s.  Every row also
checks the GPU bytes against Pillow's.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepviewagg_b200 import ops  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("unknown", "unknown")
    return name, power


def write_images(d, n, w, h, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    paths = []
    for i in range(n):
        base = 127 + 100 * np.sin(xx / (37.0 + i)) * np.cos(yy / (23.0 + i))
        img = np.clip(base[..., None] + rng.normal(0, 8, (h, w, 3)), 0, 255).astype(np.uint8)
        p = os.path.join(d, f"{w}x{h}_{i}.png")
        Image.fromarray(img).save(p, compress_level=1)
        paths.append(p)
    return paths


def algorithmic_bytes(n, w, h, wo, ho):
    """input rows the passes read + 2 x uint8 temporary (write + read) + output"""
    yb, _ = ops.resample_axis_tables(h, 0, h, ho)
    rows = int(yb[-1, 0] + yb[-1, 1] - yb[0, 0])
    return n * 3 * (rows * w + 2 * rows * wo + ho * wo)


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


def run(tag, paths, size, reps, mask=False):
    n = len(paths)
    t0 = time.perf_counter()
    arrays = [np.asarray(Image.open(p).convert("RGB")) for p in paths]
    decode_ms = (time.perf_counter() - t0) * 1e3
    h, w = arrays[0].shape[:2]
    staged = torch.empty((n, h, w, 3), dtype=torch.uint8, pin_memory=True)
    for i, a in enumerate(arrays):
        staged[i].numpy()[...] = a
    h2d_ms = time_events(lambda: staged.to("cuda", non_blocking=True), 5)
    x = staged.cuda().permute(0, 3, 1, 2)
    kernel_ms = time_events(lambda: ops.image_resample(x, size), reps)
    out = ops.image_resample(x, size)
    threads = os.cpu_count()
    ims = [Image.fromarray(a) for a in arrays]
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as pool:
        ref = list(pool.map(lambda im: np.asarray(im.resize(size)), ims))
    pillow_ms = (time.perf_counter() - t0) * 1e3
    exact = bool(np.array_equal(out.permute(0, 2, 3, 1).cpu().numpy(), np.stack(ref)))
    nbytes = algorithmic_bytes(n, w, h, size[0], size[1])
    row = dict(workload=tag, images=n, native=[w, h], out=list(size), decode_ms=round(decode_ms, 2),
               h2d_ms=round(h2d_ms, 3), kernel_ms=round(kernel_ms, 4), pillow_resize_ms=round(pillow_ms, 2),
               pillow_threads=threads, algorithmic_bytes=nbytes,
               hbm_share=round(nbytes / HBM_BYTES_PER_S * 1e3 / kernel_ms, 3), bit_exact=exact)
    if mask:
        row["mask_kernel_ms"] = round(time_events(lambda: ops.nonstatic_mask(out), reps), 4)
        m = ops.nonstatic_mask(out)
        ref_m = torch.from_numpy(np.stack(ref)).permute(0, 3, 1, 2)
        row["mask_exact"] = bool(torch.equal(m.cpu(), (ref_m[1:] != ref_m[:1]).all(dim=1).any(dim=0).t()))
        mb = n * 3 * size[0] * size[1] + size[0] * size[1]
        row["mask_hbm_share"] = round(mb / HBM_BYTES_PER_S * 1e3 / row["mask_kernel_ms"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_images.jsonl")
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_images measures on a CUDA device"
    name, power = card()
    rows = []
    with tempfile.TemporaryDirectory() as d:
        s3dis = write_images(d, 8, 4096, 2048, 0)
        kitti = write_images(d, 16, 1408, 376, 1)
        rows.append(run("s3dis_load", s3dis, (1024, 512), args.reps))
        rows.append(run("s3dis_mask", s3dis[:5], (2048, 1024), args.reps, mask=True))
        rows.append(run("kitti_load", kitti, (704, 188), args.reps))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            r.update(gpu=name, power_limit=power, torch=torch.__version__)
            f.write(json.dumps(r) + "\n")
            print(json.dumps(r))


if __name__ == "__main__":
    main()
