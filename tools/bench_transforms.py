"""Per-sample image transforms (core/multimodal/transforms.py) on an S3DIS-like synthetic sample: CUDA
containers against the same transforms on CPU containers, one JSON line per transform.

    python tools/bench_transforms.py [--out profiles/h100_transforms.jsonl] [--runs 20]

Sample: ~200 k points, 60 equirectangular uint8 images of 1024 x 512 x 3, ~8 views per point, 1 pixel per
view (exact splatting) with a 2 x 2 footprint for one view in four.  Every transform is timed by the wall
clock around a synchronised call (its host synchronisations are part of its cost): median over --runs runs
after warm-up, on fresh copies of its input.  The CPU column is the package's CPU path on the host's cores
(printed).  For the feature-map remap, achieved bytes/s (2 x output bytes / time) is reported as a fraction
of Tensor.copy_ on the same byte count, in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deepviewagg_b200 import _lib, ops  # noqa: E402
from deepviewagg_b200.core.multimodal import transforms as T  # noqa: E402
from deepviewagg_b200.core.multimodal.image import ImageMapping, SameSettingImageData  # noqa: E402


def synthetic_sample(seed=0, n_points=200_000, n_img=60, size=(1024, 512), views_per_point=8, channels=3):
    """(data, images) on the CPU: clustered footprints, one image in three straddling the x seam."""
    g = torch.Generator().manual_seed(seed)
    W, H = size
    per_img = n_points * views_per_point // n_img
    pid, iid, pix = [], [], []
    for i in range(n_img):
        k = int(per_img * (0.5 + torch.rand(1, generator=g).item()))
        pts = torch.randperm(n_points, generator=g)[:k]
        cx = 0.0 if i % 3 == 0 else float(torch.rand(1, generator=g)) * W
        cy = (0.2 + 0.6 * float(torch.rand(1, generator=g))) * H
        sx, sy = 8 + float(torch.rand(1, generator=g)) * W / 8, 4 + float(torch.rand(1, generator=g)) * H / 6
        x = torch.remainder(torch.round(cx + sx * torch.randn(k, generator=g)), W).long()
        y = torch.round(cy + sy * torch.randn(k, generator=g)).clamp(0, H - 2).long()
        big = torch.arange(k) % 4 == 0                                       # 2 x 2 footprints
        dx, dy = torch.tensor([0, 1, 0, 1]), torch.tensor([0, 0, 1, 1])
        pid += [pts, pts[big].repeat_interleave(3)]
        iid += [torch.full((k,), i), torch.full((int(big.sum()) * 3,), i)]
        pix += [torch.stack([x, y], 1),
                torch.stack([(x[big].view(-1, 1) + dx[1:]) % W, y[big].view(-1, 1) + dy[1:]], 2).view(-1, 2)]
    pid, iid, pix = torch.cat(pid), torch.cat(iid), torch.cat(pix).short()
    feat = torch.randn(pid.shape[0], 2, generator=g)
    m = ImageMapping.from_dense(pid, iid, pix, feat, num_points=n_points)
    xs = (torch.arange(W).view(1, 1, 1, W) * 5 + torch.arange(H).view(1, 1, H, 1) * 3
          + torch.arange(channels).view(1, channels, 1, 1) * 50 + torch.arange(n_img).view(n_img, 1, 1, 1) * 7)
    x = (xs % 256).to(torch.uint8)
    pos = torch.zeros(n_img, 3, dtype=torch.float64)
    pos[:, 0] = torch.arange(n_img)
    images = SameSettingImageData(pos=pos, opk=torch.zeros(n_img, 3), ref_size=size, x=x, mappings=m)
    sel = torch.randperm(n_points, generator=g)[:int(0.9 * n_points)]
    data = types.SimpleNamespace(pos=torch.zeros(sel.shape[0], 3), mapping_index=sel)
    return data, images


def chain(k_coverage=2, credit=1024 * 512 * 12):
    return [("SelectMappingFromPointId", T.SelectMappingFromPointId()),
            ("CenterRoll", T.CenterRoll(angular_res=16)),
            ("PickImagesFromMappingArea", T.PickImagesFromMappingArea(area_ratio=0.02, n_max=40, use_bbox=True)),
            ("CropImageGroups", T.CropImageGroups(padding=8, min_size=64)),
            ("PickImagesFromMemoryCredit", T.PickImagesFromMemoryCredit(credit=credit, k_coverage=k_coverage)),
            ("JitterMappingFeatures", T.JitterMappingFeatures()),
            ("RandomHorizontalFlip", T.RandomHorizontalFlip(p=1.0))]


def _to(data, images, device):
    d = types.SimpleNamespace(**{k: v.to(device) if isinstance(v, torch.Tensor) else v
                                 for k, v in vars(data).items()})
    return d, images.to(device)


def _copy(data, images):
    d = types.SimpleNamespace(**{k: v.clone() if isinstance(v, torch.Tensor) else v for k, v in vars(data).items()})
    return d, images.clone()


class _SyncCounter:
    """counts the synchronising CUDA calls (torch.cuda.set_sync_debug_mode warns on each one)"""

    def __enter__(self):
        import warnings
        self._cm = warnings.catch_warnings(record=True)
        self._log = self._cm.__enter__()
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        return self

    def __exit__(self, *exc):
        torch.cuda.set_sync_debug_mode("default")
        self._cm.__exit__(*exc)
        self.n = sum("synchroniz" in str(w.message) for w in self._log)


def _median_time(fn, inputs, runs, cuda):
    ts = []
    for inp in inputs[:runs]:
        if cuda:
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(*inp)
        if cuda:
            torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_transforms.jsonl"))
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--cpu-runs", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_transforms measures the CUDA path: it needs a GPU"
    dev = torch.device("cuda")
    props = torch.cuda.get_device_properties(0)
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        power = "unknown"
    cores = torch.get_num_threads()
    print(f"gpu {props.name}, power limit {power}, cpu threads {cores}")
    data0, images0 = synthetic_sample()
    rows = []
    # inputs of every step: the chain run once on the CPU
    stage_cpu = [(data0, images0)]
    np.random.seed(0)
    torch.manual_seed(0)
    for name, t in chain():
        d, im = _copy(*stage_cpu[-1])
        stage_cpu.append(t(d, im))
    for s, (name, t) in enumerate(chain()):
        base = stage_cpu[s]
        gpu_in = _to(*base, dev)
        warm = [_copy(*gpu_in) for _ in range(3)]
        for inp in warm:
            np.random.seed(1)
            t(*inp)
        torch.cuda.synchronize()
        inputs = [_copy(*gpu_in) for _ in range(args.runs)]
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        inp = _copy(*gpu_in)
        torch.cuda.synchronize()
        with _SyncCounter() as sc:
            np.random.seed(1)
            t(*inp)
        torch.cuda.synchronize()
        syncs = sc.n
        launches = _lib.launch_count() - n0
        np.random.seed(1)
        t_gpu = _median_time(t, inputs, args.runs, True)
        del inputs
        cpu_inputs = [_copy(*base) for _ in range(args.cpu_runs)]
        t_cpu = _median_time(t, cpu_inputs, args.cpu_runs, False)
        row = dict(transform=name, gpu=props.name, power_limit=power, cpu_threads=cores, runs=args.runs,
                   cuda_ms=round(t_gpu * 1e3, 3), cpu_ms=round(t_cpu * 1e3, 3), host_syncs=syncs,
                   native_launches=launches, n_views_in=base[1].num_views if hasattr(base[1], "num_views") else None)
        rows.append(row)
        print(json.dumps(row))
        torch.cuda.empty_cache()

    # feature-map remap against Tensor.copy_ on the same bytes
    x = images0.x.to(dev)
    B, C, H, W = x.shape
    offs = torch.stack([torch.randint(0, W - 512, (B,)), torch.randint(0, H - 256, (B,))], 1).to(dev)
    rolls = torch.randint(0, W, (B,)).to(dev)
    cases = {"roll_nchw_u8": lambda: ops.image_remap(x, rolls=rolls),
             "crop512x256_nchw_u8": lambda: ops.image_remap(x, (256, 512), offsets=offs),
             "flip_nchw_u8": lambda: ops.image_remap(x, flip=True)}
    xf = x.float().contiguous(memory_format=torch.channels_last)
    cases["roll_cl_f32"] = lambda: ops.image_remap(xf, rolls=rolls)
    cases["flip_cl_f32"] = lambda: ops.image_remap(xf, flip=True)
    for name, fn in cases.items():
        out = fn()
        nbytes = out.numel() * out.element_size()
        src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        dst = torch.empty_like(src)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        for _ in range(5):
            fn(); dst.copy_(src)
        torch.cuda.synchronize()
        reps = 50
        ev[0].record()
        for _ in range(reps):
            fn()
        ev[1].record()
        for _ in range(reps):
            dst.copy_(src)
        ev[2].record()
        torch.cuda.synchronize()
        t_k = ev[0].elapsed_time(ev[1]) / reps * 1e-3
        t_c = ev[1].elapsed_time(ev[2]) / reps * 1e-3
        row = dict(kernel="dva_image_remap", case=name, gpu=props.name, power_limit=power, bytes_moved=2 * nbytes,
                   kernel_us=round(t_k * 1e6, 2), copy_us=round(t_c * 1e6, 2),
                   kernel_GBps=round(2 * nbytes / t_k / 1e9, 1), copy_GBps=round(2 * nbytes / t_c / 1e9, 1),
                   fraction_of_copy=round(t_c / t_k, 3))
        rows.append(row)
        print(json.dumps(row))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
