"""Image loading (SameSettingImageData.read_images / load, LoadImages, NonStaticMask) on CPU containers against
the fixtures executed on the reference (tests/golden/images_load.npz), the numpy restatement of Pillow's resize
(oracle/image_resample_oracle.py) against the installed Pillow, and the new container state (`path`, `mask`)
through indexing, clone, to, batching and storage.  The check_* helpers take a device and are shared with
tests/test_gpu_images.py."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import GOLDEN
from deepviewagg_b200 import ops
from deepviewagg_b200.core.multimodal import transforms as T
from deepviewagg_b200.core.multimodal.image import ImageMapping, SameSettingImageBatch, SameSettingImageData
from deepviewagg_b200.core.multimodal.storage import load_image_data, save_image_data
from oracle import image_resample_oracle as O


def fixture():
    return np.load(os.path.join(GOLDEN, "images_load.npz"), allow_pickle=False)


def write_pngs(z, directory):
    """the fixture's PNG bytes -> {setting: [paths]}"""
    paths = {}
    for k in ("equi", "persp"):
        paths[k] = []
        for i in range(int(z[f"png/{k}/count"])):
            p = os.path.join(str(directory), f"{k}_{i}.png")
            with open(p, "wb") as f:
                f.write(z[f"png/{k}/{i}"].tobytes())
            paths[k].append(p)
    return paths


def container(paths, device, **kw):
    n = len(paths)
    return SameSettingImageData(pos=torch.zeros(n, 3, device=device), path=np.array(paths, dtype=object), **kw)


def read_case_tags(z):
    return sorted({k.split("/")[1] for k in z.files if k.startswith("read/")})


def check_read(device, tmp_path):
    z = fixture()
    paths = write_pngs(z, tmp_path)
    for tag in read_case_tags(z):
        pre = f"read/{tag}/"
        im = container(paths[str(z[pre + "setting"])], device)
        kw = dict(size=tuple(z[pre + "size"].tolist()))
        if tag == "idx_subset":
            kw["idx"] = torch.from_numpy(z[pre + "idx"])
        for key in ("rollings", "crop_offsets"):
            if pre + key in z.files:
                kw[key] = torch.from_numpy(z[pre + key])
        if pre + "crop_size" in z.files:
            kw["crop_size"] = tuple(z[pre + "crop_size"].tolist())
        if pre + "downscale" in z.files:
            kw["downscale"] = float(z[pre + "downscale"])
        x = im.read_images(**kw)
        assert x.device.type == torch.device(device).type and x.dtype == torch.uint8, tag
        assert x.stride() == tuple(z[pre + "stride"].tolist()), tag
        assert torch.equal(x.cpu(), torch.from_numpy(z[pre + "x"])), tag


def check_load(device, tmp_path):
    z = fixture()
    paths = write_pngs(z, tmp_path)
    im = container(paths["equi"], device, ref_size=(80, 40))
    im.rollings = torch.from_numpy(z["load/rollings"]).to(device)
    loader = T.LoadImages(ref_size=tuple(z["load/ref_size"].tolist()), crop_size=tuple(z["load/crop_size"].tolist()),
                          crop_offsets=torch.from_numpy(z["load/crop_offsets"]).to(device),
                          downscale=float(z["load/downscale"]))
    _, im = loader(None, im)
    assert im.x.device.type == torch.device(device).type
    assert im.img_size == tuple(z["load/img_size"].tolist())
    assert torch.equal(im.x.cpu(), torch.from_numpy(z["load/x"]))


def mask_tags(z):
    return sorted({k.split("/")[1] for k in z.files if k.startswith("mask/")})


def check_mask(device, tmp_path):
    z = fixture()
    paths = write_pngs(z, tmp_path)
    for tag in mask_tags(z):
        pre = f"mask/{tag}/"
        ref_size = tuple(z[pre + "ref_size"].tolist())
        im = container(paths[str(z[pre + "setting"])], device, ref_size=ref_size, proj_upscale=2)
        torch.manual_seed(int(z[pre + "seed"]))
        _, im = T.NonStaticMask(ref_size=ref_size, proj_upscale=2, n_sample=int(z[pre + "n_sample"]))(None, im)
        assert im.mask.dtype == torch.bool and tuple(im.mask.shape) == im.proj_size
        assert im.mask.device.type == torch.device(device).type
        assert torch.equal(im.mask.cpu(), torch.from_numpy(z[pre + "mask"])), tag


# ------------------------------------------------------------------------------------------------
# the oracle against Pillow and against the fixtures
# ------------------------------------------------------------------------------------------------
RESIZE_CASES = [
    ((256, 128), (64, 32), None), ((256, 128), (128, 64), None), ((97, 61), (40, 23), None),
    ((200, 100), (50, 25), None), ((50, 30), (73, 41), None), ((50, 30), (100, 60), None), ((31, 17), (1, 1), None),
    ((31, 17), (31, 1), None), ((31, 17), (1, 17), None), ((64, 48), (37, 48), None), ((64, 48), (64, 13), None),
    ((64, 48), (20, 15), (3.5, 2.25, 40.75, 30.5)), ((64, 48), (30, 20), (0, 0, 64, 48)),
    ((64, 48), (10, 10), (10, 5, 30, 25)), ((64, 48), (32, 24), (32, 24, 64, 48)), ((64, 48), (64, 48), (1, 1, 64, 48)),
    ((33, 17), (100, 3), (0.1, 0, 33, 16.9)), ((80, 40), (41, 20), (7, 3, 77, 37)),
]


@pytest.mark.parametrize("src,size,box", RESIZE_CASES)
def test_oracle_equals_pillow(src, size, box):
    img = np.random.default_rng(hash((src, size)) % 2**32).integers(0, 256, (src[1], src[0], 3), dtype=np.uint8)
    ref = np.asarray(Image.fromarray(img).resize(size, box=box))
    assert np.array_equal(O.resize(img, size, box), ref)


@pytest.mark.parametrize("src,size,box", RESIZE_CASES)
def test_host_tables_equal_oracle_coefficients(src, size, box):
    """ops.resample_axis_tables (vectorised, what the kernel consumes) == the oracle's per-index restatement"""
    b = box or (0, 0) + src
    for n_in, c0, c1, n_out in ((src[0], b[0], b[2], size[0]), (src[1], b[1], b[3], size[1])):
        ob, ok = O.coefficients(n_in, c0, c1, n_out)
        vb, vk = ops.resample_axis_tables(n_in, c0, c1, n_out)
        assert np.array_equal(ob, vb) and np.array_equal(ok, vk)


def test_fixture_records_pillow_version():
    import PIL
    assert str(fixture()["pillow_version"]) == PIL.__version__


def test_oracle_reproduces_fixture_reads(tmp_path):
    """the reference's read_images == decode + oracle resize + roll + crop / box resize"""
    z = fixture()
    paths = write_pngs(z, tmp_path)
    for tag in read_case_tags(z):
        pre = f"read/{tag}/"
        size = tuple(z[pre + "size"].tolist())
        idx = z[pre + "idx"]
        rolls = z[pre + "rollings"] if pre + "rollings" in z.files else np.zeros(len(idx), dtype=np.int64)
        crop = tuple(z[pre + "crop_size"].tolist()) if pre + "crop_size" in z.files else size
        offs = z[pre + "crop_offsets"] if pre + "crop_offsets" in z.files else np.zeros((len(idx), 2), dtype=np.int64)
        down = float(z[pre + "downscale"]) if pre + "downscale" in z.files else None
        out = []
        for i, r, (left, top) in zip(idx, rolls, offs):
            a = np.asarray(Image.open(paths[str(z[pre + "setting"])][i]).convert("RGB"))
            a = np.roll(O.resize(a, size), -int(r), axis=1)
            if down is None:
                a = a[top:top + crop[1], left:left + crop[0]]
            else:
                end = tuple(int(v / down) for v in crop)
                a = O.resize(a, end, (left, top, left + crop[0], top + crop[1]))
            out.append(a)
        assert np.array_equal(np.stack(out).transpose(0, 3, 1, 2), z[pre + "x"]), tag


# ------------------------------------------------------------------------------------------------
# CPU containers against the fixtures
# ------------------------------------------------------------------------------------------------
def test_read_images_cpu(tmp_path):
    check_read("cpu", tmp_path)


def test_load_images_cpu(tmp_path):
    check_load("cpu", tmp_path)


def test_nonstatic_mask_cpu(tmp_path):
    check_mask("cpu", tmp_path)


def test_nonstatic_mask_draw_quirk():
    """image 0 has weight 0: it is drawn only when every image is, and then last (the fixture pins the same)"""
    z = fixture()
    for tag in mask_tags(z):
        drawn = z[f"mask/{tag}/drawn"].tolist()
        n = int(z[f"png/{z[f'mask/{tag}/setting']}/count"])
        if drawn:
            assert (0 in drawn) == (len(drawn) == n)
            if 0 in drawn:
                assert drawn[-1] == 0


# ------------------------------------------------------------------------------------------------
# container state: path and mask
# ------------------------------------------------------------------------------------------------
def _toy(n=4, mask=True):
    pix = torch.tensor([[1, 2], [3, 4], [5, 6], [7, 1]], dtype=torch.int16)
    maps = ImageMapping.from_dense(torch.tensor([0, 1, 2, 3]), torch.tensor([0, 1, 2, 3]) % n, pix, None,
                                   num_points=4)
    im = SameSettingImageData(pos=torch.arange(3 * n, dtype=torch.float64).view(n, 3), ref_size=(8, 4),
                              proj_upscale=2, path=np.array([f"img_{i}.png" for i in range(n)], dtype=object),
                              x=torch.arange(n * 3 * 4 * 8, dtype=torch.uint8).view(n, 3, 4, 8), mappings=maps)
    if mask:
        m = torch.zeros(16, 8, dtype=torch.bool)
        m[3:9, 2:] = True
        im.mask = m
    return im


def test_path_and_mask_through_indexing_clone_to_batching():
    im = _toy()
    assert im.proj_size == (16, 8)
    sub = im[[2, 0]]
    assert sub.path.tolist() == ["img_2.png", "img_0.png"]
    assert torch.equal(sub.mask, im.mask) and sub.mask.data_ptr() != im.mask.data_ptr()
    c = im.clone()
    assert c.path.tolist() == im.path.tolist() and torch.equal(c.mask, im.mask)
    t = im.to("cpu")
    assert t.path.tolist() == im.path.tolist() and torch.equal(t.mask, im.mask)
    other = _toy(mask=False)
    other.mask = ~im.mask
    assert other.settings_hash == im.settings_hash           # the mask is not a setting of the hash
    b = SameSettingImageBatch.from_data_list([im, other])
    assert b.path.tolist() == im.path.tolist() + other.path.tolist()
    assert torch.equal(b.mask, im.mask)                       # the first item's mask serves the batch
    assert SameSettingImageBatch.from_data_list([_toy(mask=False), im]).mask is None


def test_storage_round_trip_with_x_mask_path(tmp_path):
    im = _toy()
    im._x = im.x.contiguous(memory_format=torch.channels_last)
    f = save_image_data(os.path.join(str(tmp_path), "s.dva"), im)
    back = load_image_data(f)[0]
    assert back.path.tolist() == im.path.tolist()
    assert torch.equal(back.mask, im.mask)
    assert torch.equal(back.x, im.x) and back.x.stride() == im.x.stride()
    plain = _toy(mask=False)
    plain.path = None
    back = load_image_data(save_image_data(os.path.join(str(tmp_path), "p.dva"), plain))[0]
    assert back.mask is None and back.path is None and back.x.stride() == plain.x.stride()
    assert torch.equal(back.x, plain.x)


def test_argument_errors(tmp_path):
    z = fixture()
    paths = write_pngs(z, tmp_path)
    im = container(paths["equi"], "cpu")
    with pytest.raises(AssertionError):
        im.mask = torch.ones(5, 5, dtype=torch.bool)              # not proj_size
    with pytest.raises(AssertionError):
        im.mask = torch.ones(im.proj_size, dtype=torch.uint8)     # not bool
    with pytest.raises(AssertionError):
        im.read_images(size=(40, 20), crop_size=(20, 10))         # crop_size without crop_offsets
    with pytest.raises(AssertionError):
        im.read_images(size=(40, 20), rollings=torch.zeros(6, dtype=torch.int32))
    with pytest.raises(AssertionError):
        im.read_images(size=(40, 20), rollings=torch.zeros(5, dtype=torch.long))
    with pytest.raises(AssertionError):
        im.read_images(size=(40, 20), crop_size=(50, 10), crop_offsets=torch.zeros(6, 2, dtype=torch.long))
    with pytest.raises(AssertionError):
        im.read_images(size=(40, 20), crop_size=(30, 10), crop_offsets=torch.full((6, 2), 15, dtype=torch.long))
    with pytest.raises(AssertionError):
        im.read_images(size=(40, 20), downscale=0.5)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        ops.image_resample(torch.zeros(1, 3, 4, 4, dtype=torch.uint8), (2, 2))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        ops.nonstatic_mask(torch.zeros(2, 3, 4, 4, dtype=torch.uint8))


def test_entry_points_validate_arguments():
    """no launch: argument checks of the C entry points"""
    from deepviewagg_b200 import _lib
    lib = _lib.load()
    assert lib.dva_resample_u8(None, None, None, -1, 4, 4, 3, 2, 2, 2, None, None, 5, 0, None, None, 5, 0, None,
                               None) == _lib.DVA_EINVAL
    assert lib.dva_resample_u8(None, None, None, 1, 4, 4, 5, 2, 2, 2, None, None, 5, 0, None, None, 5, 0, None,
                               None) == _lib.DVA_EUNSUPPORTED
    assert lib.dva_resample_u8(None, None, None, 1, 4, 4, 3, 2, 2, 2, None, None, 5, 0, None, None, 5, 0, None,
                               None) == _lib.DVA_EINVAL                     # neither pass
    assert b"resample_u8" in lib.dva_last_error()
    assert lib.dva_nonstatic_mask(None, 1, 4, 4, 3, None, None) == _lib.DVA_EINVAL
    assert lib.dva_nonstatic_mask(None, 2, 4, 4, 3, None, None) == _lib.DVA_EINVAL
    assert b"nonstatic_mask" in lib.dva_last_error()
