"""Image transforms on CUDA containers: the fixtures executed on the reference, bit for bit; the remap
kernel against torch slicing / roll / flip; the statistics kernel against scatter_reduce; the coverage
kernels against the CPU path; the whole chain on CUDA against the CPU chain, then one UnimodalBranch step."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import ROOT
from deepviewagg_b200 import ops
from deepviewagg_b200.core.multimodal import transforms as T
from deepviewagg_b200.core.multimodal.image import ImageData
from test_transforms import check_chain, check_memory_credit, check_quantisation, check_ties

sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_transforms import chain, synthetic_sample  # noqa: E402

pytestmark = pytest.mark.gpu


def test_chain_fixture_cuda():
    check_chain("cuda")


def test_center_roll_quantisation_cuda():
    check_quantisation("cuda")


def test_area_ties_cuda():
    check_ties("cuda")


def test_memory_credit_fixture_cuda():
    check_memory_credit("cuda")


def _remap_ref(x, Ho, Wo, rolls, offsets, flip):
    out = []
    for b in range(x.shape[0]):
        im = x[b]
        if rolls is not None:
            im = torch.roll(im, int(rolls[b]), dims=-1)
        if offsets is not None:
            ox, oy = int(offsets[b, 0]), int(offsets[b, 1])
            im = im[:, oy:oy + Ho, ox:ox + Wo]
        if flip:
            im = torch.flip(im, dims=[-1])
        out.append(im)
    return torch.stack(out)


@pytest.mark.parametrize("dtype", [torch.uint8, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("channels_last", [False, True])
def test_image_remap_against_torch(dtype, channels_last):
    g = torch.Generator().manual_seed(0)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    for (B, C, H, W) in ((5, 3, 17, 33), (4, 8, 16, 64), (3, 1, 9, 255), (2, 4, 32, 1024)):
        if dtype == torch.uint8:
            x = torch.randint(0, 256, (B, C, H, W), generator=g, dtype=torch.uint8)
        else:
            x = torch.randn(B, C, H, W, generator=g).to(dtype)
        xg = x.cuda().contiguous(memory_format=fmt)
        # rolls 0, 1, W - 1 and random
        rolls = torch.tensor(([0, W - 1, 1] + torch.randint(0, W, (B,), generator=g).tolist())[:B])
        out = ops.image_remap(xg, rolls=rolls.cuda())
        assert out.is_contiguous(memory_format=fmt)
        assert torch.equal(out.cpu(), _remap_ref(x, H, W, rolls, None, False)), ("roll", B, C, H, W)
        # crops: offsets at both borders and odd sizes
        for Ho, Wo in ((H, W), (H - 1, W - 3), (max(1, H // 2), max(1, W // 2) | 1), (1, 1)):
            ox = torch.tensor(([0, W - Wo] + torch.randint(0, W - Wo + 1, (B,), generator=g).tolist())[:B])
            oy = torch.tensor(([H - Ho, 0] + torch.randint(0, H - Ho + 1, (B,), generator=g).tolist())[:B])
            offs = torch.stack([ox, oy], 1)
            out = ops.image_remap(xg, (Ho, Wo), offsets=offs.cuda())
            assert out.is_contiguous(memory_format=fmt)
            assert torch.equal(out.cpu(), _remap_ref(x, Ho, Wo, None, offs, False)), ("crop", B, C, H, W, Ho, Wo)
            out = ops.image_remap(xg, (Ho, Wo), rolls=rolls.cuda(), offsets=offs.cuda(), flip=True)
            assert torch.equal(out.cpu(), _remap_ref(x, Ho, Wo, rolls, offs, True)), ("all", B, C, H, W, Ho, Wo)
        out = ops.image_remap(xg, flip=True)
        assert torch.equal(out.cpu(), torch.flip(x, dims=[-1])), ("flip", B, C, H, W)


@pytest.mark.parametrize("pix_dtype", [torch.int16, torch.int32, torch.int64])
def test_mapping_image_stats_against_scatter_reduce(pix_dtype):
    """1 M random views, some with hundreds of pixels, and images without any pixel"""
    g = torch.Generator().manual_seed(1)
    V, n_img, ref_w, H = 1_000_000, 300, 1000, 500
    images = torch.randint(0, n_img, (V,), generator=g)
    images[(images % 7) == 3] = 5                              # images 3, 10, ... are empty; 5 is crowded
    counts = torch.randint(0, 4, (V,), generator=g)
    counts[torch.randint(0, V, (50,), generator=g)] = 700       # many-pixel views
    aptr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)])
    P = int(aptr[-1])
    pix = torch.stack([torch.randint(0, ref_w, (P,), generator=g), torch.randint(0, H, (P,), generator=g)], 1)
    pix = pix.to(pix_dtype)
    count, bbox, occ = ops.mapping_image_stats(images.cuda(), aptr.cuda(), pix.cuda(), n_img, ref_w=ref_w)
    idx = images.repeat_interleave(counts)
    assert torch.equal(count.cpu(), torch.bincount(idx, minlength=n_img))
    i2 = idx.view(-1, 1).expand(-1, 2)
    p64 = pix.long()
    mn = torch.zeros((n_img, 2), dtype=torch.long).scatter_reduce(0, i2, p64, 'amin', include_self=False)
    mx = torch.zeros((n_img, 2), dtype=torch.long).scatter_reduce(0, i2, p64, 'amax', include_self=False)
    ref = torch.stack([mn[:, 0], mx[:, 0], mn[:, 1], mx[:, 1]], 1)
    assert (count.cpu() == 0).sum() > 10
    assert torch.equal(bbox.cpu().long(), ref)
    q = (p64[:, 0].float() * 256 / ref_w).long() & 255
    dense = torch.zeros((n_img, 256), dtype=torch.bool)
    dense[idx, q] = True
    bits = torch.zeros((n_img, 8), dtype=torch.long)
    for k in range(8):
        for b in range(32):
            bits[:, k] |= dense[:, 32 * k + b].long() << b
    assert torch.equal(occ.cpu().long() & 0xFFFFFFFF, bits)


def test_coverage_picks_cuda_equal_cpu():
    """200 k points, 60 images over 3 settings, 5 seeds"""
    from test_transforms import make_images
    g = torch.Generator().manual_seed(2)
    N = 200_000
    settings = []
    for k, (n_img, size) in enumerate(((20, (1024, 512)), (25, (512, 256)), (15, (256, 128)))):
        pid, iid = [], []
        for i in range(n_img):
            kk = int(torch.randint(5000, 40000, (1,), generator=g))
            pid.append(torch.randperm(N, generator=g)[:kk])
            iid.append(torch.full((kk,), i))
        pid, iid = torch.cat(pid), torch.cat(iid)
        pix = torch.stack([torch.randint(0, size[0], pid.shape, generator=g),
                           torch.randint(0, size[1], pid.shape, generator=g)], 1).short()
        settings.append(dict(point_ids=pid, image_ids=iid, pixels=pix, features=torch.zeros(pid.shape[0], 1),
                             n_img=n_img, size=size))

    def build(device):
        return ImageData([make_images(s, s["n_img"], s["size"], N, device=device) for s in settings])
    cpu_in = build("cpu")
    for seed in range(5):
        picks = {}
        for device in ("cpu", "cuda"):
            images = cpu_in.clone() if device == "cpu" else cpu_in.to("cuda")
            np.random.seed(seed)
            _, out = T.PickImagesFromMemoryCredit(credit=1024 * 512 * 6, k_coverage=2)(
                types.SimpleNamespace(num_nodes=N), images)
            picks[device] = [(tuple(im.ref_size), im.pos[:, 0].long().cpu().tolist()) for im in out]
        assert picks["cpu"] == picks["cuda"], seed
        assert sum(len(p) for _, p in picks["cpu"]) >= 5


def _same(a, b):
    la = list(a) if isinstance(a, ImageData) else [a]
    lb = list(b) if isinstance(b, ImageData) else [b]
    assert len(la) == len(lb)
    for x, y in zip(la, lb):
        assert x.crop_size == y.crop_size
        assert torch.equal(x.pos.cpu(), y.pos.cpu())
        assert torch.equal(x.rollings.cpu(), y.rollings.cpu())
        assert (x.crop_offsets is None) == (y.crop_offsets is None)
        if x.crop_offsets is not None:
            assert torch.equal(x.crop_offsets.cpu(), y.crop_offsets.cpu())
        assert torch.equal(x.x.cpu(), y.x.cpu())
        mx, my = x.mappings, y.mappings
        for t, u in ((mx.pointers, my.pointers), (mx.images, my.images), (mx.values[1].pointers, my.values[1].pointers),
                     (mx.pixels, my.pixels), (mx.features, my.features)):
            assert t.dtype == u.dtype and torch.equal(t.cpu(), u.cpu())


def test_whole_chain_cuda_equals_cpu_then_branch_step():
    from deepviewagg_b200.modules.multimodal.fusion import BimodalFusion
    from deepviewagg_b200.modules.multimodal.modules import UnimodalBranch
    from deepviewagg_b200.modules.multimodal.pooling import BimodalCSRPool
    data, images = synthetic_sample(seed=3)
    results = {}
    for device in ("cpu", "cuda"):
        d = types.SimpleNamespace(pos=data.pos.to(device), mapping_index=data.mapping_index.to(device))
        im = images.clone().to(device)
        torch.manual_seed(5)
        np.random.seed(5)
        for _, t in chain():
            d, im = t(d, im)
        results[device] = (d, im)
    _same(results["cpu"][1], results["cuda"][1])
    d, mod = results["cuda"]
    assert isinstance(mod, ImageData) and mod.num_settings >= 2
    xs = []
    for im in mod:
        x = (im.x.float() / 255).requires_grad_(True)
        im._x = x
        xs.append(x)
    n = d.pos.shape[0]
    branch = UnimodalBranch(None, BimodalCSRPool("max"), BimodalCSRPool("mean"), BimodalFusion("concatenation"),
                            out_channels=6).cuda()
    x_3d = torch.randn(n, 3, device="cuda", requires_grad=True)
    out = branch({"x_3d": x_3d, "x_seen": None, "modalities": {"image": mod}}, "image")
    assert out["x_3d"].shape[0] == n and torch.isfinite(out["x_3d"]).all()
    grads = torch.autograd.grad(out["x_3d"].square().sum(), [x_3d] + xs)
    assert all(torch.isfinite(gr).all() for gr in grads)
    assert any(float(gr.abs().sum()) > 0 for gr in grads[1:])
