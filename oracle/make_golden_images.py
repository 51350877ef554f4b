"""Generate the image-loading fixtures by EXECUTING THE REFERENCE (oracle; test infrastructure).

Run in the build container only (needs the reference checkout, see oracle/ref_loader.py):
    PYTORCH_JIT=0 python -m oracle.make_golden_images
writes tests/golden/images_load.npz and tests/golden/visibility_model_masked.npz with the saver of
oracle/make_golden.py:

- images_load: seeded PNGs (stored as bytes) of two settings: equirectangular-shaped images with a band of
  pixels identical across images (a camera rig) plus a region where only one channel is shared, and small
  perspective images.  The reference's SameSettingImageData.read_images for several (size, rollings, crop,
  downscale) combinations, including fractional-ratio downscale boxes and an upscale, its load(), and
  NonStaticMask._process under fixed torch seeds.
- visibility_model_masked: SplattingVisibility.__call__ on the numba path with a banded img_mask.
"""
import io
import os
import sys
import tempfile

os.environ.setdefault("PYTORCH_JIT", "0")

import numpy as np  # noqa: E402
import PIL  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import save  # noqa: E402


def make_pngs(seed=3):
    """-> {setting: [png bytes]}: 'equi' 6 images 160 x 80 (rows 64.. identical, a block sharing only the red
    channel), 'persp' 3 images 70 x 45.  Smooth fields plus noise, so that resampling mixes distinct values."""
    rng = np.random.default_rng(seed)
    out = {}
    yy, xx = np.mgrid[0:80, 0:160]
    rig = rng.integers(0, 256, (16, 160, 3), dtype=np.uint8)
    red = rng.integers(0, 256, (24, 32), dtype=np.uint8)
    equi = []
    for i in range(6):
        base = 127 + 100 * np.sin(xx / (7.0 + i) + i)[..., None] * np.cos(yy / (5.0 + 2 * i))[..., None]
        img = np.clip(base + rng.normal(0, 25, (80, 160, 3)), 0, 255).astype(np.uint8)
        img[64:] = rig
        img[8:32, 120:152, 0] = red
        equi.append(img)
    out["equi"] = equi
    out["persp"] = [rng.integers(0, 256, (45, 70, 3), dtype=np.uint8) for _ in range(3)]
    pngs = {}
    for k, imgs in out.items():
        pngs[k] = []
        for img in imgs:
            buf = io.BytesIO()
            Image.fromarray(img).save(buf, format="PNG")
            pngs[k].append(buf.getvalue())
    return pngs


def write_pngs(pngs, directory):
    paths = {}
    for k, blobs in pngs.items():
        paths[k] = []
        for i, b in enumerate(blobs):
            p = os.path.join(directory, f"{k}_{i}.png")
            with open(p, "wb") as f:
                f.write(b)
            paths[k].append(p)
    return paths


# (tag, setting, read_images kwargs); rollings / crop offsets are drawn from a seeded generator in main()
READ_CASES = [
    ("plain", "equi", dict(size=(80, 40))),
    ("native", "persp", dict(size=(70, 45))),
    ("quarter", "equi", dict(size=(40, 20))),
    ("odd", "equi", dict(size=(73, 41))),
    ("one_px", "persp", dict(size=(1, 1))),
    ("upscale", "persp", dict(size=(113, 64))),
    ("roll_crop", "equi", dict(size=(80, 40), roll=True, crop=(60, 30))),
    ("roll_down2", "equi", dict(size=(80, 40), roll=True, crop=(60, 30), downscale=2)),
    ("crop_down_frac", "equi", dict(size=(96, 48), roll=True, crop=(70, 34), downscale=1.7)),
    ("persp_down_frac", "persp", dict(size=(70, 45), crop=(51, 33), downscale=2.5)),
    ("idx_subset", "equi", dict(size=(48, 24), idx=[4, 1, 2], roll=True)),
]


def main():
    ref = ref_loader.load_reference()
    T = ref_loader.load_transforms()
    SSID = ref.image.SameSettingImageData
    pngs = make_pngs()
    arrays = {"pillow_version": np.array(PIL.__version__)}
    for k, blobs in pngs.items():
        arrays[f"png/{k}/count"] = np.array(len(blobs))
        for i, b in enumerate(blobs):
            arrays[f"png/{k}/{i}"] = np.frombuffer(b, dtype=np.uint8)
    gen = torch.Generator().manual_seed(11)
    with tempfile.TemporaryDirectory() as d:
        paths = write_pngs(pngs, d)

        def container(k, **kw):
            n = len(paths[k])
            return SSID(path=np.array(paths[k]), pos=torch.zeros(n, 3), **kw)

        for tag, k, c in READ_CASES:
            im = container(k)
            idx = np.array(c["idx"]) if "idx" in c else np.arange(len(paths[k]))
            n, size = len(idx), c["size"]
            kw = dict(idx=torch.from_numpy(idx) if "idx" in c else None, size=size)
            if c.get("roll"):
                kw["rollings"] = torch.randint(-2 * size[0], 2 * size[0], (n,), generator=gen)
            if "crop" in c:
                cw, ch = c["crop"]
                kw["crop_size"] = (cw, ch)
                kw["crop_offsets"] = torch.stack([torch.randint(0, size[0] - cw + 1, (n,), generator=gen),
                                                  torch.randint(0, size[1] - ch + 1, (n,), generator=gen)], 1)
            if "downscale" in c:
                kw["downscale"] = c["downscale"]
            x = im.read_images(**kw)
            print(tag, tuple(x.shape), x.stride())
            arrays[f"read/{tag}/setting"] = np.array(k)
            arrays[f"read/{tag}/idx"] = idx
            arrays[f"read/{tag}/size"] = np.array(size)
            for key in ("rollings", "crop_offsets"):
                if key in kw:
                    arrays[f"read/{tag}/{key}"] = kw[key]
            if "crop_size" in kw:
                arrays[f"read/{tag}/crop_size"] = np.array(kw["crop_size"])
            if "downscale" in kw:
                arrays[f"read/{tag}/downscale"] = np.array(float(kw["downscale"]))
            arrays[f"read/{tag}/x"] = x.contiguous()
            arrays[f"read/{tag}/stride"] = np.array(x.stride())

        # load(): the container's own state, through LoadImages
        im = container("equi", ref_size=(80, 40))
        im.rollings = torch.tensor([0, 7, -13, 99, 250, 3])
        loader = T.LoadImages(ref_size=(80, 40), crop_size=(56, 29),
                              crop_offsets=torch.tensor([[0, 0], [24, 11], [5, 1], [12, 7], [23, 10], [1, 2]]),
                              downscale=1.4)
        _, im = loader(None, im)
        arrays.update({"load/ref_size": np.array((80, 40)), "load/crop_size": np.array((56, 29)),
                       "load/crop_offsets": loader.crop_offsets, "load/downscale": np.array(1.4),
                       "load/rollings": im.rollings, "load/x": im.x.contiguous(),
                       "load/img_size": np.array(im.img_size)})
        print("load", tuple(im.x.shape))

        # NonStaticMask: torch.manual_seed(seed) right before the call; n_sample < n, == n, and < 2
        for tag, k, n_sample, seed in (("n3", "equi", 3, 0), ("n6", "equi", 6, 1), ("n4_s5", "equi", 4, 5),
                                       ("persp_n2", "persp", 2, 2), ("n1", "equi", 1, 0)):
            im = container(k, ref_size=(80, 40) if k == "equi" else (35, 22), proj_upscale=2)
            torch.manual_seed(seed)
            _, im = T.NonStaticMask(ref_size=im.ref_size, proj_upscale=2, n_sample=n_sample)(None, im)
            torch.manual_seed(seed)
            drawn = torch.multinomial(torch.arange(len(paths[k]), dtype=torch.float), min(n_sample, len(paths[k]))) \
                if min(n_sample, len(paths[k])) >= 2 else torch.zeros(0, dtype=torch.long)
            arrays.update({f"mask/{tag}/setting": np.array(k), f"mask/{tag}/n_sample": np.array(n_sample),
                           f"mask/{tag}/seed": np.array(seed), f"mask/{tag}/ref_size": np.array(im.ref_size),
                           f"mask/{tag}/drawn": drawn, f"mask/{tag}/mask": im.mask})
            print("mask", tag, tuple(im.mask.shape), int(im.mask.sum()), drawn.tolist())
    save("images_load", **arrays)
    make_masked_visibility(ref)


def make_masked_visibility(ref):
    """SplattingVisibility.__call__ (visibility.py:1677-1776) with an img_mask: masked pixels drop their points
    before the splat (field_of_view, visibility.py:428-434).  Same scene as visibility_model_equirect_exact."""
    gen = torch.Generator().manual_seed(29)
    n = 7000
    xyz = (torch.rand(n, 3, generator=gen) - 0.5) * torch.tensor([12., 12., 4.])
    geo = torch.rand(n, 3, generator=gen)
    normals = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=1)
    img_xyz = torch.tensor([0.3, -0.2, 0.1])
    ctor = dict(voxel=0.05, exact=True, img_size=(512, 256), crop_top=16, crop_bottom=24, r_max=8, r_min=0.5,
                camera="s3dis_equirectangular")
    mask = torch.ones(512, 256, dtype=torch.bool)
    mask[:, 170:] = False                 # a rig band at the bottom
    mask[300:360] = False                 # and a vertical strip
    call = dict(img_opk=torch.tensor([0.05, -0.1, 0.7]), img_mask=mask)
    model = ref.visibility.SplattingVisibility(**ctor)
    out = model(xyz, img_xyz, linearity=geo[:, 0], planarity=geo[:, 1], scattering=geo[:, 2], normals=normals,
                **call)
    unmasked = model(xyz, img_xyz, linearity=geo[:, 0], planarity=geo[:, 1], scattering=geo[:, 2], normals=normals,
                     img_opk=call["img_opk"])
    print("masked splat", tuple(out["idx"].shape), "unmasked", tuple(unmasked["idx"].shape))
    save("visibility_model_masked", xyz=xyz, img_xyz=img_xyz, geo=geo, normals=normals,
         ctor_keys=np.array(list(ctor.keys())), **{"ctor/" + k: np.asarray(v) for k, v in ctor.items()},
         **{"call/" + k: v for k, v in call.items()}, **{"out/" + k: v for k, v in out.items()})


if __name__ == "__main__":
    main()
