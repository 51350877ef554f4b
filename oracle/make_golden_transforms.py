"""Generate the image-transform fixtures by EXECUTING THE REFERENCE (oracle; test infrastructure).

Run in the build container only (needs the reference checkout, see oracle/ref_loader.py):
    PYTORCH_JIT=0 python -m oracle.make_golden_transforms
writes tests/golden/transforms_{chain,quantisation,ties,memory_credit}.npz with the saver of
oracle/make_golden.py.  The reference transforms (core/data_transform/multimodal/image.py) run on the
CPU with the torch_scatter stand-in.  Every image carries its id in pos[:, 0], so the images a step keeps
are read back from `pos` ("ids", in output order).  The reference's SameSettingImageData.__getitem__
resets `rollings` to zeros, so rollings are recorded right after CenterRoll only.  To keep the files small,
the input maps (the closed formula of image_x) are stored as shape and sum only, the chain stores `x` and the
mapping features after CropImageGroups and after the last step, and the CenterRoll-only fixture has no maps.
"""
import os
import sys

os.environ.setdefault("PYTORCH_JIT", "0")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import save  # noqa: E402


def synthetic_sample(seed, n_points, n_img, ref_size, per_img=(150, 400), seam_every=3, n_feat=2):
    """Clustered pixel footprints on equirectangular images; every third cluster straddles the x seam.
    Returns the dense (point, image, pixel, feature) items (one per (point, image) pair) and a uint8 x."""
    g = np.random.default_rng(seed)
    W, H = ref_size
    pid, iid, pix = [], [], []
    for i in range(n_img):
        k = int(g.integers(*per_img))
        pts = g.choice(n_points, size=k, replace=False)
        cx = 0.0 if i % seam_every == 0 else g.uniform(0, W)
        cy = g.uniform(0.2 * H, 0.8 * H)
        sx, sy = g.uniform(3, W / 8), g.uniform(2, H / 6)
        x = np.mod(np.rint(cx + sx * g.standard_normal(k)), W).astype(np.int64)
        y = np.clip(np.rint(cy + sy * g.standard_normal(k)), 0, H - 1).astype(np.int64)
        pid.append(pts)
        iid.append(np.full(k, i))
        pix.append(np.stack([x, y], 1))
    pid, iid, pix = np.concatenate(pid), np.concatenate(iid), np.concatenate(pix)
    feat = g.standard_normal((pid.shape[0], n_feat)).astype(np.float32)
    return dict(point_ids=pid, image_ids=iid, pixels=pix.astype(np.int16), features=feat)


def image_x(n_img, C, H, W):
    """x[i, c, y, w] = (7 i + 50 c + 3 y + 5 w + (y w mod 11)) mod 256, uint8"""
    i, c, y, w = np.meshgrid(np.arange(n_img), np.arange(C), np.arange(H), np.arange(W), indexing="ij")
    return ((7 * i + 50 * c + 3 * y + 5 * w + (y * w) % 11) % 256).astype(np.uint8)


def ref_images(ref, s, n_img, ref_size, N, x=None, with_features=True):
    I = ref.image
    m = I.ImageMapping.from_dense(torch.from_numpy(s["point_ids"]), torch.from_numpy(s["image_ids"]),
                                  torch.from_numpy(s["pixels"]),
                                  torch.from_numpy(s["features"]) if with_features else None, num_points=N)
    pos = torch.zeros(n_img, 3, dtype=torch.float64)
    pos[:, 0] = torch.arange(n_img)
    return I.SameSettingImageData(path=np.array([f"{i}" for i in range(n_img)], dtype="O"), pos=pos,
                                  opk=torch.zeros(n_img, 3), ref_size=ref_size,
                                  x=torch.from_numpy(x) if x is not None else None, mappings=m)


def state(prefix, images, with_x=True, with_features=True):
    """fields of every setting of an ImageData (or one SameSettingImageData) under prefix/<k>/"""
    items = list(images) if not isinstance(images, ref_loader.load_reference().image.SameSettingImageData) \
        else [images]
    out = {prefix + "/n_settings": np.array(len(items))}
    for k, im in enumerate(items):
        m = im.mappings
        p = f"{prefix}/{k}/"
        out.update({p + "ids": im.pos[:, 0].long(), p + "crop_size": np.array(im.crop_size),
                    p + "crop_offsets": im.crop_offsets, p + "pointers": m.pointers, p + "images": m.images,
                    p + "atomic_pointers": m.values[1].pointers, p + "pixels": m.pixels})
        if with_features and m.has_features:
            out[p + "features"] = m.features
        if with_x and im.x is not None:
            out[p + "x"] = im.x
    # copies: later transforms update the containers in place (CenterRoll writes the pixels)
    return {k: v.clone() if isinstance(v, torch.Tensor) else v for k, v in out.items()}


def _integer_scatter(standin):
    """scatter_min / scatter_max of the stand-in for integer sources (the transforms reduce uint8 widths and
    int16 pixels): reduced in float64 (exact for these ranges), cast back; an empty segment gives 0 as in torch_scatter."""
    import types

    def wrap(fn):
        def f(src, index, dim=0, **kw):
            if src.dtype.is_floating_point:
                return fn(src, index, dim=dim, **kw)
            vals, arg = fn(src.double(), index, dim=dim, **kw)
            return vals.to(src.dtype), arg
        return f
    ns = types.SimpleNamespace(**{k: getattr(standin, k) for k in dir(standin) if not k.startswith("__")})
    ns.scatter_min, ns.scatter_max = wrap(standin.scatter_min), wrap(standin.scatter_max)
    return ns


def make_data_cls(ref):
    T = ref_loader.load_transforms()
    T.torch_scatter = ref.image.torch_scatter = _integer_scatter(sys.modules["torch_scatter"])
    base = ref.Data

    class Data(base):
        def __getitem__(self, k):
            return getattr(self, k)

        def __setitem__(self, k, v):
            setattr(self, k, v)

        def clone(self):
            return Data(**{k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in self.__dict__.items()})
    return T, Data


def make_chain(ref):
    T, Data = make_data_cls(ref)
    N, n_img, ref_size, n_sel = 2000, 24, (256, 128), 1500
    s = synthetic_sample(1, N, n_img, ref_size)
    x = image_x(n_img, 3, ref_size[1], ref_size[0])
    sel = np.random.default_rng(2).permutation(N)[:n_sel]
    images = ref_images(ref, s, n_img, ref_size, N, x=x)
    data = Data(pos=torch.rand(n_sel, 3, generator=torch.Generator().manual_seed(3)),
                mapping_index=torch.from_numpy(sel))
    kw = dict(area_ratio=0.01, n_max=18, padding=4, min_size=16, credit=64 * 64 * 9, k_coverage=2,
              sigma=0.02, clip=0.03, angular_res=16, seed=7)
    torch.manual_seed(kw["seed"])
    np.random.seed(kw["seed"])
    arrays = dict(**s, x0_shape=np.array(x.shape), x0_sum=np.array(x.sum(dtype=np.int64)), mapping_index=sel,
                  N=np.array(N), ref_size=np.array(ref_size), kw=repr(kw))
    chain = [("select", T.SelectMappingFromPointId()), ("roll", T.CenterRoll(angular_res=kw["angular_res"])),
             ("area", T.PickImagesFromMappingArea(area_ratio=kw["area_ratio"], n_max=kw["n_max"], use_bbox=True)),
             ("crop", T.CropImageGroups(padding=kw["padding"], min_size=kw["min_size"])),
             ("credit", T.PickImagesFromMemoryCredit(credit=kw["credit"], k_coverage=kw["k_coverage"])),
             ("jitter", T.JitterMappingFeatures(sigma=kw["sigma"], clip=kw["clip"]))]
    for name, t in chain:
        data, images = t(data, images)
        changed = name in ("crop", "jitter")          # the steps that rebuild the mappings / change x or features
        arrays.update(state(name, images, with_x=changed, with_features=changed))
        if name == "roll":
            arrays["roll/rollings"] = images.rollings
        print(name, images)
    save("transforms_chain", **arrays)


def make_quantisation(ref):
    """CenterRoll at ref_W = 250: the fp32 quantisation and the roll rounding are not exact there"""
    T, Data = make_data_cls(ref)
    N, n_img, ref_size = 900, 20, (250, 120)
    s = synthetic_sample(5, N, n_img, ref_size, per_img=(20, 120), seam_every=2)
    arrays = dict(**s, n_img=np.array(n_img), N=np.array(N), ref_size=np.array(ref_size))
    for ar in (16, 3):
        images = ref_images(ref, s, n_img, ref_size, N)
        _, images = T.CenterRoll(angular_res=ar)(Data(pos=torch.zeros(N, 3)), images)
        arrays.update(state(f"ar{ar}", images))
        arrays[f"ar{ar}/rollings"] = images.rollings
    save("transforms_quantisation", **arrays)


def make_ties(ref):
    """PickImagesFromMappingArea with tied areas straddling n_max: boxes of w x h with equal products, and
    equal pixel counts"""
    T, Data = make_data_cls(ref)
    n_img, ref_size = 12, (128, 64)
    dims = [(10, 6), (6, 10), (12, 5), (15, 4), (20, 3), (10, 6), (30, 2), (4, 15), (8, 8), (16, 4), (2, 30), (5, 12)]
    pid, iid, pix = [], [], []
    p = 0
    for i, (w, h) in enumerate(dims):
        xs = np.array([3, 3 + w, 3 + w // 2, 3 + w // 3, 3 + (2 * w) // 3])         # 5 pixels per image
        ys = np.array([1, 1 + h, 1 + h // 2, 1 + (2 * h) // 3, 1 + h // 3])
        pid.append(np.arange(p, p + 5))
        iid.append(np.full(5, i))
        pix.append(np.stack([xs, ys], 1))
        p += 5
    s = dict(point_ids=np.concatenate(pid), image_ids=np.concatenate(iid),
             pixels=np.concatenate(pix).astype(np.int16),
             features=np.zeros((p, 1), dtype=np.float32))
    arrays = dict(**s, N=np.array(p), ref_size=np.array(ref_size))
    for tag, kw in (("bbox5", dict(area_ratio=0.001, n_max=5, use_bbox=True)),
                    ("bbox9", dict(area_ratio=0.005, n_max=9, use_bbox=True)),
                    ("count4", dict(area_ratio=0.0001, n_max=4, use_bbox=False)),
                    ("none", dict(area_ratio=0.5, n_max=4, n_min=1, use_bbox=True))):
        images = ref_images(ref, s, n_img, ref_size, p)
        _, out = T.PickImagesFromMappingArea(**kw)(Data(pos=torch.zeros(p, 3)), images)
        arrays[tag + "/ids"] = out.pos[:, 0].long()
        arrays.update({f"{tag}/{k}": np.array(v) for k, v in kw.items()})
    save("transforms_ties", **arrays)


def make_memory_credit(ref):
    """PickImagesFromMemoryCredit over 4 settings of different image sizes sharing the same points,
    k_coverage 0 and 2, seeds 0..4"""
    T, Data = make_data_cls(ref)
    N = 3000
    sizes = [(64, 32), (32, 32), (128, 64), (64, 64)]
    counts = [9, 14, 6, 8]
    arrays = dict(N=np.array(N), n_settings=np.array(len(sizes)))
    samples = []
    for k, (sz, n) in enumerate(zip(sizes, counts)):
        s = synthetic_sample(20 + k, N, n, sz, per_img=(100, 900))
        samples.append(s)
        arrays.update({f"in/{k}/{f}": v for f, v in s.items()})
        arrays[f"in/{k}/ref_size"] = np.array(sz)
    credit = 64 * 32 * 12
    arrays["credit"] = np.array(credit)
    for kc in (0, 2):
        for seed in range(5):
            images = ref.image.ImageData([ref_images(ref, s, n, sz, N) for s, sz, n in zip(samples, sizes, counts)])
            np.random.seed(seed)
            _, out = T.PickImagesFromMemoryCredit(credit=credit, k_coverage=kc)(Data(pos=torch.zeros(N, 3)), images)
            p = f"k{kc}/seed{seed}"
            arrays[p + "/n_settings"] = np.array(out.num_settings)
            for j, im in enumerate(out):
                arrays[f"{p}/{j}/ids"] = im.pos[:, 0].long()
                arrays[f"{p}/{j}/ref_size"] = np.array(im.ref_size)
    save("transforms_memory_credit", **arrays)


if __name__ == "__main__":
    ref = ref_loader.load_reference()
    ref_loader.load_transforms()
    make_chain(ref)
    make_quantisation(ref)
    make_ties(ref)
    make_memory_credit(ref)
