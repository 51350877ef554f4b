"""Image loading on CUDA containers: dva_resample_u8 bit-exact against the numpy restatement of Pillow's resize,
read_images / load / LoadImages / NonStaticMask equal to the fixtures executed on the reference byte for byte,
the masked SplattingVisibility against its reference fixture, masked MapImages against the per-image oracle
pipeline, and the pre_transform chain LoadImages -> NonStaticMask -> MapImages ->
NeighborhoodBasedMappingFeatures on CUDA containers against the same chain loaded on CPU containers."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import GOLDEN, load_golden
from deepviewagg_b200 import ops
from deepviewagg_b200.core.multimodal import transforms as T
from deepviewagg_b200.core.multimodal.image import SameSettingImageData
from deepviewagg_b200.core.multimodal.mapping import MapImages, NeighborhoodBasedMappingFeatures
from oracle import image_resample_oracle as O
from oracle import visibility_oracle as VO
from test_images import RESIZE_CASES, check_load, check_mask, check_read

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("src,size,box", RESIZE_CASES)
def test_resample_kernel_equals_oracle(src, size, box):
    rng = np.random.default_rng(7)
    imgs = rng.integers(0, 256, (3, src[1], src[0], 3), dtype=np.uint8)
    x = torch.from_numpy(imgs).cuda().permute(0, 3, 1, 2)
    out = ops.image_resample(x, size, boxes=box)
    assert out.shape == (3, 3, size[1], size[0])
    assert out.stride() == (size[0] * size[1] * 3, 1, size[0] * 3, 3)          # channels-last, like the reference
    ref = np.stack([O.resize(a, size, box) for a in imgs]).transpose(0, 3, 1, 2)
    assert np.array_equal(out.cpu().numpy(), ref)


def test_resample_kernel_per_image_boxes():
    """one launch, a different box per image (integer, fractional, touching the borders)"""
    rng = np.random.default_rng(8)
    imgs = rng.integers(0, 256, (5, 90, 160, 3), dtype=np.uint8)
    boxes = [(0, 0, 120, 60), (40, 30, 160, 90), (3.5, 2.25, 100.75, 70.5), (17, 11, 137, 71), (0.5, 0, 160, 89.5)]
    out = ops.image_resample(torch.from_numpy(imgs).cuda().permute(0, 3, 1, 2), (52, 27),
                             boxes=torch.tensor(boxes, dtype=torch.float32))
    ref = np.stack([O.resize(a, (52, 27), b) for a, b in zip(imgs, boxes)]).transpose(0, 3, 1, 2)
    assert np.array_equal(out.cpu().numpy(), ref)
    # and a list input in NCHW memory
    lst = [torch.from_numpy(a).cuda().permute(2, 0, 1).contiguous() for a in imgs[:2]]
    out = ops.image_resample(lst, (40, 20))
    ref = np.stack([O.resize(a, (40, 20)) for a in imgs[:2]]).transpose(0, 3, 1, 2)
    assert np.array_equal(out.cpu().numpy(), ref)


def test_nonstatic_mask_kernel_equals_torch():
    g = torch.Generator().manual_seed(3)
    imgs = torch.randint(0, 4, (5, 3, 37, 53), generator=g, dtype=torch.uint8)
    ref = (imgs[1:] != imgs[:1]).all(dim=1).any(dim=0).t()
    got = ops.nonstatic_mask(imgs.cuda().contiguous(memory_format=torch.channels_last))
    assert got.shape == (53, 37) and torch.equal(got.cpu(), ref)


def test_read_images_cuda(tmp_path):
    check_read("cuda", tmp_path)


def test_load_images_cuda(tmp_path):
    check_load("cuda", tmp_path)


def test_nonstatic_mask_cuda(tmp_path):
    check_mask("cuda", tmp_path)


def test_read_images_cuda_chunks(tmp_path):
    """a byte budget smaller than one image and mixed native sizes: one chunk per run of equal size"""
    rng = np.random.default_rng(9)
    paths = []
    for i, (w, h) in enumerate([(64, 32), (64, 32), (50, 30), (64, 32), (50, 30), (50, 30)]):
        p = os.path.join(str(tmp_path), f"{i}.png")
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(p)
        paths.append(p)
    cpu = SameSettingImageData(pos=torch.zeros(6, 3), path=np.array(paths, dtype=object))
    gpu = cpu.to("cuda")
    gpu._READ_CHUNK_BYTES = 1
    kw = dict(size=(40, 22), rollings=torch.tensor([0, 5, -3, 41, 7, 1]), crop_size=(30, 17),
              crop_offsets=torch.tensor([[0, 0], [10, 5], [3, 2], [1, 1], [9, 4], [5, 0]]), downscale=1.3)
    assert torch.equal(gpu.read_images(**kw).cpu(), cpu.read_images(**kw))
    kw.pop("downscale")
    assert torch.equal(gpu.read_images(**kw).cpu(), cpu.read_images(**kw))


def test_masked_splatting_visibility_vs_reference():
    from deepviewagg_b200.core.multimodal import visibility as V
    z = np.load(os.path.join(GOLDEN, "visibility_model_masked.npz"))
    ctor = {k: (z["ctor/" + k].tolist() if z["ctor/" + k].ndim else z["ctor/" + k].item())
            for k in z["ctor_keys"].tolist()}
    ctor["img_size"] = tuple(ctor["img_size"])
    call = {k[5:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("call/")}
    call["img_mask"] = call["img_mask"].cuda()
    ref = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("out/")}
    geo = torch.from_numpy(z["geo"]).cuda()
    out = V.SplattingVisibility(**ctor)(torch.from_numpy(z["xyz"]).cuda(), torch.from_numpy(z["img_xyz"]),
                                        linearity=geo[:, 0], planarity=geo[:, 1], scattering=geo[:, 2],
                                        normals=torch.from_numpy(z["normals"]).cuda(), **call)
    for k in ("idx", "x", "y", "depth"):
        assert out[k].dtype == ref[k].dtype and torch.equal(out[k].cpu(), ref[k]), k
    assert (out["features"].cpu() - ref["features"]).abs().max() <= 1e-6


def _scene():
    g = load_golden("zbuffer_nocrop")
    W, H = [int(v) for v in g["size"]]
    cams = torch.stack([g["img_xyz"], g["img_xyz"] + torch.tensor([1.5, -0.7, 0.1])])
    opk = torch.stack([g["img_opk"], g["img_opk"] * 0.5])
    return g["xyz"], cams, opk, W, H


def _mapping_equal(a, b):
    assert torch.equal(a.pointers.cpu(), b.pointers.cpu())
    assert torch.equal(a.images.cpu(), b.images.cpu())
    assert torch.equal(a.values[1].pointers.cpu(), b.values[1].pointers.cpu())
    assert a.pixels.dtype == b.pixels.dtype and torch.equal(a.pixels.cpu(), b.pixels.cpu())
    assert torch.equal(a.features.cpu(), b.features.cpu())


def test_map_images_all_true_mask_is_no_mask():
    xyz, cams, opk, W, H = _scene()
    plain = SameSettingImageData(pos=cams, opk=opk, ref_size=(W // 2, H // 2), proj_upscale=2)
    masked = SameSettingImageData(pos=cams, opk=opk, ref_size=(W // 2, H // 2), proj_upscale=2,
                                  mask=torch.ones(W, H, dtype=torch.bool))
    a = MapImages(voxel=0.05, exact=True, r_max=8, r_min=0.5)(xyz, plain)
    b = MapImages(voxel=0.05, exact=True, r_max=8, r_min=0.5)(xyz, masked)
    _mapping_equal(a.mappings, b.mappings)
    assert torch.equal(b.mask.cpu(), masked.mask)


def test_map_images_banded_mask_equals_oracle():
    """MapImages with a mask == per-image C-oracle projection, mask filter, splat z-buffer, numpy from_dense"""
    xyz, cams, opk, W, H = _scene()
    mask = torch.ones(W, H, dtype=torch.bool)
    mask[:, int(H * 0.7):] = False
    mask[W // 3: W // 2] = False
    images = SameSettingImageData(pos=cams, opk=opk, ref_size=(W // 2, H // 2), proj_upscale=2, mask=mask)
    out = MapImages(voxel=0.05, exact=True, r_max=8, r_min=0.5)(xyz, images)
    m = out.mappings
    mk = mask.numpy()
    pid, iid, pix = [], [], []
    for i in range(2):
        R = VO.pose_to_rotation_matrix(opk[i].numpy())
        dist, xp, yp, keep = VO.project_equirect(xyz.numpy(), cams[i].numpy(), R, W, H, 0, 0, 0.5, 8.0)
        idx = np.where(keep)[0]
        idx = idx[mk[np.floor(xp[idx]).astype(np.int64), np.floor(yp[idx]).astype(np.int64)]]
        sp = VO.splat_boxes(xp[idx], yp[idx], dist[idx], W, H, voxel=0.05)
        i2, x2, y2, _ = VO.zbuffer(sp, dist[idx], xp[idx], yp[idx], W, H, exact=True)
        p, x, y = idx[i2], x2 // 2, y2 // 2
        u = VO.lexargunique(p, x, y)
        pid.append(p[u]); iid.append(np.full(len(u), i)); pix.append(np.stack([x[u], y[u]], 1))
    ref = VO.image_mapping_from_dense(np.concatenate(pid), np.concatenate(iid), np.concatenate(pix), None,
                                      xyz.shape[0])
    assert np.array_equal(m.pointers.cpu().numpy(), ref["pointers"])
    assert np.array_equal(m.images.cpu().numpy(), ref["images"])
    assert np.array_equal(m.atomic_csr_indexing.cpu().numpy(), ref["atomic_pointers"])
    assert np.array_equal(m.pixels.cpu().numpy().astype(np.int64), ref["pixels"])
    plain = SameSettingImageData(pos=cams, opk=opk, ref_size=(W // 2, H // 2), proj_upscale=2)
    assert MapImages(voxel=0.05, exact=True, r_max=8, r_min=0.5)(xyz, plain).mappings.num_items > m.num_items


def test_pre_transform_chain_cuda_equals_cpu(tmp_path):
    """LoadImages -> NonStaticMask -> MapImages -> NeighborhoodBasedMappingFeatures, S3DIS-like scene: the
    first two steps on CUDA containers give the same x, mask and mappings as on CPU containers"""
    xyz, cams, opk, W, H = _scene()
    rng = np.random.default_rng(12)
    rig = rng.integers(0, 256, (H // 4, W, 3), dtype=np.uint8)
    paths = []
    for i in range(2):
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        img[-H // 4:] = rig
        p = os.path.join(str(tmp_path), f"{i}.png")
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="PNG")
        open(p, "wb").write(buf.getvalue())
        paths.append(p)
    results = []
    for dev in ("cpu", "cuda"):
        images = SameSettingImageData(pos=cams.to(dev), opk=opk.to(dev), path=np.array(paths, dtype=object))
        _, images = T.LoadImages(ref_size=(W // 2, H // 2))(None, images)
        torch.manual_seed(0)
        _, images = T.NonStaticMask(ref_size=(W // 2, H // 2), proj_upscale=2, n_sample=5)(None, images)
        assert images.x.device.type == dev and images.mask.device.type == dev
        images = MapImages(voxel=0.05, exact=True, r_max=8, r_min=0.5)(xyz, images)
        images = NeighborhoodBasedMappingFeatures(k=[10, 20])(xyz, images.to("cuda"))
        results.append(images)
    a, b = results
    assert not bool(a.mask.all()) and bool(a.mask.any())
    assert torch.equal(a.x.cpu(), b.x.cpu()) and torch.equal(a.mask.cpu(), b.mask.cpu())
    _mapping_equal(a.mappings, b.mappings)
