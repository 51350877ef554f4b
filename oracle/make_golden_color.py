"""Generate the colour-transform fixtures by EXECUTING THE REFERENCE (oracle; test infrastructure).

Run in the build container only (needs the reference checkout and torchvision, see oracle/ref_loader.py):
    PYTORCH_JIT=0 python -m oracle.make_golden_color
writes tests/golden/color_jitter.npz and tests/golden/color_float.npz with the saver of oracle/make_golden.py.
The reference's ColorJitter, ToFloatImage, Normalize and ToImageData (core/data_transform/multimodal/image.py:64-68,
:1221-1283) run on the CPU with the installed torchvision, on one thread so that torch.mean is reproducible.  The
inputs follow the closed formulas of oracle/color_oracle.color_input and are stored as shape and sum only.  For
every ColorJitter step the fixture records the drawn fn_idx and factors (NaN: off), and for the contrast op the
mean torch.mean gave (recorded by wrapping torchvision's adjust_contrast) and the exact mean of the same image.
Seeds are taken from 0 upwards until all 6 relative orders of brightness, contrast and saturation occur for the
S3DIS and the KITTI-360 factors.  The large case (one 512 x 1024 image, where torch's fp32 mean is inexact) stores
the SHA-256 of its output instead of the output.
"""
import hashlib
import os
import sys

os.environ.setdefault("PYTORCH_JIT", "0")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import color_oracle as O  # noqa: E402
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import save  # noqa: E402

S3DIS, KITTI = (0.6, 0.6, 0.7), (0.2, 0.2, 0.2)      # s3disfused-sparse.yaml, kitti360-sparse*.yaml
SHAPE = (3, 61, 97)                                  # B, H, W: odd sizes
KINDS = ("formula", "edges", "ramps")


def order_seeds(cfg):
    """the first seeds whose draws give each of the 6 relative orders of ops 0, 1, 2"""
    ranges = [O.check_input(v) for v in cfg]
    seen, seeds, seed = set(), [], 0
    while len(seen) < 6:
        torch.manual_seed(seed)
        fn_idx = O.draw(*ranges)[0]
        order = tuple(int(i) for i in fn_idx if int(i) < 3)
        if order not in seen:
            seen.add(order)
            seeds.append(seed)
        seed += 1
    return seeds


class Recorder:
    """wraps torchvision's ColorJitter.get_params and adjust_contrast to record the draws and the means"""

    def __init__(self):
        import torchvision.transforms as TV
        import torchvision.transforms._functional_tensor as FT
        import torchvision.transforms.functional as F
        self.TV, self.FT, self.F = TV, FT, F
        self.draws, self.means = [], []
        get_params, adjust_contrast = TV.ColorJitter.get_params, F.adjust_contrast

        def rec_params(*a):
            out = get_params(*a)
            self.draws.append(out)
            return out

        def rec_contrast(img, factor):
            g = FT.rgb_to_grayscale(img)
            self.means.append((torch.mean(g.to(torch.float32), dim=(-3, -2, -1)).numpy().reshape(-1),
                               O.exact_mean(g[:, 0].numpy())))
            return adjust_contrast(img, factor)
        TV.ColorJitter.get_params = staticmethod(rec_params)
        F.adjust_contrast = rec_contrast


class _Data:
    """the `data` argument: the reference's ImageData dispatch clones it once per setting"""

    def clone(self):
        return self


def container(ref, x):
    n = x.shape[0]
    return ref.image.SameSettingImageData(path=np.array([f"{i}" for i in range(n)], dtype="O"),
                                          pos=torch.zeros(n, 3, dtype=torch.float64), opk=torch.zeros(n, 3),
                                          ref_size=(x.shape[3], x.shape[2]), x=torch.from_numpy(x))


def run_jitter(ref, RT, rec, name, cfg, seed, settings, out, store_out=True):
    """settings: list of (kind, B, H, W); one ImageData when there are several"""
    xs = [O.color_input(k, B, H, W) for k, B, H, W in settings]
    ims = [container(ref, x) for x in xs]
    images = ims[0] if len(ims) == 1 else ref.image.ImageData(ims)
    rec.draws.clear()
    rec.means.clear()
    torch.manual_seed(seed)
    _, res = RT.ColorJitter(*cfg)(_Data(), images)
    res = [res] if len(ims) == 1 else list(res)
    assert len(rec.draws) == len(ims)
    p = f"jitter/{name}/"
    out.update({p + "config": np.array(cfg), p + "seed": np.array(seed), p + "n_settings": np.array(len(ims))})
    means = iter(rec.means)
    for s, ((kind, B, H, W), x, r, draw) in enumerate(zip(settings, xs, res, rec.draws)):
        q = f"{p}{s}/"
        fn_idx, b, c, sat, _ = draw
        out.update({q + "kind": np.array(kind), q + "shape": np.array([B, 3, H, W]),
                    q + "input_sum": np.array(int(x.astype(np.int64).sum())), q + "fn_idx": fn_idx,
                    q + "factors": np.array([np.nan if v is None else v for v in (b, c, sat)], dtype=np.float64)})
        if c is not None:
            tm, em = next(means)
            out[q + "torch_mean"], out[q + "exact_mean"] = tm, em
        y = np.ascontiguousarray(r.x.numpy())
        if store_out:
            out[q + "out"] = y
        else:
            out[q + "out_sha256"] = np.array(hashlib.sha256(y.tobytes()).hexdigest())
    assert next(means, None) is None


def main():
    torch.set_num_threads(1)
    ref = ref_loader.load_reference()
    RT = ref_loader.load_transforms()
    rec = Recorder()
    out = {}
    for tag, cfg in (("s3dis", S3DIS), ("kitti", KITTI)):
        for j, seed in enumerate(order_seeds(cfg)):
            run_jitter(ref, RT, rec, f"{tag}_{seed}", cfg, seed, [(KINDS[j % 3],) + SHAPE], out)
    run_jitter(ref, RT, rec, "contrast_only", (0, 0.5, 0), 11, [("ramps",) + SHAPE], out)
    run_jitter(ref, RT, rec, "saturation_only", (0, 0, 0.5), 12, [("ramps",) + SHAPE], out)
    run_jitter(ref, RT, rec, "no_brightness", (0, 0.6, 0.7), 13, [("edges",) + SHAPE], out)
    run_jitter(ref, RT, rec, "two_settings", S3DIS, 14, [("formula",) + SHAPE, ("ramps", 2, 40, 33)], out)
    run_jitter(ref, RT, rec, "large", S3DIS, 3, [("formula", 1, 512, 1024)], out, store_out=False)
    save("color_jitter", **out)

    fl = {}
    x = O.color_input("edges", 3, 13, 29)
    fl.update({"float/kind": np.array("edges"), "float/shape": np.array(x.shape),
               "float/input_sum": np.array(int(x.astype(np.int64).sum()))})
    im = container(ref, x)
    _, im = RT.ToFloatImage()(None, im)
    fl["float/to_float"] = im.x.numpy().copy()
    _, im = RT.Normalize()(None, im)
    fl["float/normalize"] = im.x.numpy().copy()
    mean, std = [0.5, 0.25, 0.125], [0.3, 0.7, 0.0625]
    im = container(ref, x)
    _, im = RT.ToFloatImage()(None, im)
    _, im = RT.Normalize(mean=mean, std=std)(None, im)
    fl.update({"float/normalize_custom": im.x.numpy().copy(), "float/custom_mean": np.array(mean),
               "float/custom_std": np.array(std)})
    _, wrapped = RT.ToImageData()(None, container(ref, x))
    fl["to_image_data/n_settings"] = np.array(len(wrapped))
    fl["to_image_data/x_equal"] = np.array(bool(torch.equal(wrapped[0].x, torch.from_numpy(x))))
    save("color_float", **fl)


if __name__ == "__main__":
    main()
