"""Image transforms (core/multimodal/transforms.py) on CPU containers against fixtures executed on the
reference (oracle/make_golden_transforms.py), bit for bit; dispatch; argument checks of the C entry points.
The helpers here are shared with tests/test_gpu_transforms.py."""
import types

import numpy as np
import pytest
import torch

from conftest import load_golden
from deepviewagg_b200 import _lib
from deepviewagg_b200.core.multimodal import transforms as T
from deepviewagg_b200.core.multimodal.image import ImageData, ImageMapping, SameSettingImageData


def make_images(g, n_img, ref_size, N, x=None, prefix="", device="cpu"):
    m = ImageMapping.from_dense(g[prefix + "point_ids"], g[prefix + "image_ids"], g[prefix + "pixels"],
                                g[prefix + "features"], num_points=N)
    pos = torch.zeros(n_img, 3, dtype=torch.float64)
    pos[:, 0] = torch.arange(n_img)
    im = SameSettingImageData(pos=pos, opk=torch.zeros(n_img, 3), ref_size=tuple(ref_size), x=x, mappings=m)
    return im.to(device)


def fixture_x(g):
    """the chain fixture's input maps: x[i, c, y, w] = (7 i + 50 c + 3 y + 5 w + (y w mod 11)) mod 256, uint8
    (oracle/make_golden_transforms.py:image_x), pinned by the stored shape and sum"""
    n, C, H, W = g["x0_shape"].tolist()
    i, c, y, w = torch.meshgrid(torch.arange(n), torch.arange(C), torch.arange(H), torch.arange(W), indexing="ij")
    x = ((7 * i + 50 * c + 3 * y + 5 * w + (y * w) % 11) % 256).to(torch.uint8)
    assert int(x.long().sum()) == int(g["x0_sum"])
    return x


def _settings(images):
    return list(images) if isinstance(images, ImageData) else [images]


def check_state(g, prefix, images, rollings=None):
    """every recorded field of step `prefix` equals ours; rollings (of the CenterRoll step) follow the ids"""
    items = _settings(images)
    assert len(items) == int(g[prefix + "/n_settings"]), prefix
    for k, im in enumerate(items):
        p = f"{prefix}/{k}/"
        m = im.mappings
        ids = im.pos[:, 0].long().cpu()
        assert torch.equal(ids, g[p + "ids"]), p + "ids"
        assert tuple(im.crop_size) == tuple(g[p + "crop_size"].tolist()), p + "crop_size"
        offs = im.crop_offsets if im.crop_offsets is not None else torch.zeros((im.num_views, 2), dtype=torch.long)
        assert torch.equal(offs.cpu(), g[p + "crop_offsets"]), p + "crop_offsets"
        for f, t in (("pointers", m.pointers), ("images", m.images), ("atomic_pointers", m.values[1].pointers),
                     ("pixels", m.pixels)):
            ref = g[p + f]
            assert t.dtype == ref.dtype and torch.equal(t.cpu(), ref), p + f
        if p + "features" in g:
            assert torch.equal(m.features.cpu(), g[p + "features"]), p + "features"
        if p + "x" in g:
            assert im.x.dtype == torch.uint8 and torch.equal(im.x.cpu(), g[p + "x"]), p + "x"
        if rollings is not None:
            assert torch.equal(im.rollings.cpu(), rollings[ids]), p + "rollings"


def run_chain(g, device, check=True):
    """the fixture's chain on our containers, checked against the fixture after every step (the transforms
    update containers in place, as the reference does); returns the final (data, images)"""
    kw = g["kw"]
    N = int(g["N"])
    x0 = fixture_x(g)
    images = make_images(g, x0.shape[0], g["ref_size"].tolist(), N, x=x0, device=device)
    data = types.SimpleNamespace(pos=torch.zeros(g["mapping_index"].shape[0], 3, device=device),
                                 mapping_index=g["mapping_index"].to(device))
    torch.manual_seed(kw["seed"])
    np.random.seed(kw["seed"])
    chain = [("select", T.SelectMappingFromPointId()), ("roll", T.CenterRoll(angular_res=kw["angular_res"])),
             ("area", T.PickImagesFromMappingArea(area_ratio=kw["area_ratio"], n_max=kw["n_max"], use_bbox=True)),
             ("crop", T.CropImageGroups(padding=kw["padding"], min_size=kw["min_size"])),
             ("credit", T.PickImagesFromMemoryCredit(credit=kw["credit"], k_coverage=kw["k_coverage"])),
             ("jitter", T.JitterMappingFeatures(sigma=kw["sigma"], clip=kw["clip"]))]
    roll = g["roll/rollings"]
    for name, t in chain:
        data, images = t(data, images)
        if name == "select":
            assert torch.equal(data.mapping_index.cpu(), torch.arange(data.pos.shape[0]))
        if check:
            check_state(g, name, images, rollings=None if name == "select" else roll)
    return data, images


def check_chain(device):
    g = load_golden("transforms_chain")
    assert g["roll/rollings"].unique().numel() > 3           # the seam-straddling clusters do get rolled
    run_chain(g, device)


def check_quantisation(device):
    g = load_golden("transforms_quantisation")
    for ar in (16, 3):
        images = make_images(g, int(g["n_img"]), g["ref_size"].tolist(), int(g["N"]), device=device)
        _, images = T.CenterRoll(angular_res=ar)(types.SimpleNamespace(num_nodes=int(g["N"])), images)
        assert torch.equal(images.rollings.cpu(), g[f"ar{ar}/rollings"])
        check_state(g, f"ar{ar}", images)
    # 250 is not a power of two: some rollings are not multiples of 250 / 16
    assert (g["ar16/rollings"] % 125 != 0).any()


def check_ties(device):
    g = load_golden("transforms_ties")
    for tag in ("bbox5", "bbox9", "count4", "none"):
        kw = {k: g[f"{tag}/{k}"].item() for k in ("area_ratio", "n_max", "n_min", "use_bbox") if f"{tag}/{k}" in g}
        images = make_images(g, 12, g["ref_size"].tolist(), int(g["N"]), device=device)
        _, out = T.PickImagesFromMappingArea(**kw)(types.SimpleNamespace(num_nodes=int(g["N"])), images)
        assert torch.equal(out.pos[:, 0].long().cpu(), g[tag + "/ids"]), tag


def memory_credit_inputs(g, device):
    n_set = int(g["n_settings"])
    N = int(g["N"])
    return ImageData([make_images(g, int(g[f"in/{k}/image_ids"].max()) + 1, g[f"in/{k}/ref_size"].tolist(), N,
                                  prefix=f"in/{k}/", device=device) for k in range(n_set)])


def check_memory_credit(device):
    g = load_golden("transforms_memory_credit")
    N = int(g["N"])
    for kc in (0, 2):
        for seed in range(5):
            images = memory_credit_inputs(g, device)
            np.random.seed(seed)
            t = T.PickImagesFromMemoryCredit(credit=int(g["credit"]), k_coverage=kc)
            _, out = t(types.SimpleNamespace(num_nodes=N), images)
            p = f"k{kc}/seed{seed}"
            assert out.num_settings == int(g[p + "/n_settings"]), p
            for j, im in enumerate(out):
                assert tuple(im.ref_size) == tuple(g[f"{p}/{j}/ref_size"].tolist()), p
                assert torch.equal(im.pos[:, 0].long().cpu(), g[f"{p}/{j}/ids"]), (p, j)


# ------------------------------------------------------------------------------------------------------------
def test_chain_cpu():
    check_chain("cpu")


def test_center_roll_quantisation_cpu():
    check_quantisation("cpu")


def test_area_ties_cpu():
    check_ties("cpu")


def test_memory_credit_cpu():
    check_memory_credit("cpu")


def _tiny():
    pid = torch.tensor([0, 0, 1, 2, 2, 3])
    iid = torch.tensor([0, 1, 1, 0, 1, 1])
    pix = torch.tensor([[1, 2], [3, 4], [5, 6], [7, 1], [2, 2], [9, 3]], dtype=torch.int16)
    m = ImageMapping.from_dense(pid, iid, pix, torch.ones(6, 2), num_points=4)
    x = torch.arange(2 * 3 * 8 * 16, dtype=torch.float32).view(2, 3, 8, 16)
    return SameSettingImageData(pos=torch.zeros(2, 3), ref_size=(16, 8), x=x, mappings=m)


def test_dispatch_list_imagedata_and_process_image_data():
    jit = T.JitterMappingFeatures()
    # list: item by item
    a, b = _tiny(), _tiny()
    data = [types.SimpleNamespace(num_nodes=4), types.SimpleNamespace(num_nodes=4)]
    d_out, i_out = jit(data, [a, b])
    assert isinstance(d_out, list) and isinstance(i_out, list) and len(i_out) == 2
    # ImageData without _PROCESS_IMAGE_DATA: setting by setting, one ImageData out
    _, out = jit(types.SimpleNamespace(num_nodes=4), ImageData([_tiny(), _tiny()]))
    assert isinstance(out, ImageData) and out.num_settings == 2
    # a transform that splits a setting returns one flat ImageData
    _, out = T.CropImageGroups(min_size=4)(types.SimpleNamespace(num_nodes=4), ImageData([_tiny(), _tiny()]))
    assert isinstance(out, ImageData) and all(isinstance(im, SameSettingImageData) for im in out)
    assert out.num_views == 4
    # _PROCESS_IMAGE_DATA wraps a SameSettingImageData into an ImageData
    np.random.seed(0)
    _, out = T.PickImagesFromMemoryCredit(credit=16 * 8 * 2)(types.SimpleNamespace(num_nodes=4), _tiny())
    assert isinstance(out, ImageData) and out.num_views == 2
    # CropImageGroups on no image: ImageData of the input
    empty = _tiny()[torch.zeros(0, dtype=torch.long)]
    _, out = T.CropImageGroups()(types.SimpleNamespace(num_nodes=4), empty)
    assert isinstance(out, ImageData) and out.num_views == 0


def test_container_rollings_state():
    im = _tiny()
    assert im.rollings.dtype == torch.long and torch.equal(im.rollings, torch.zeros(2, dtype=torch.long))
    im.update_rollings(torch.tensor([3, 15]))
    assert torch.equal(im.x[1], torch.roll(_tiny().x[1], 15, dims=-1))
    assert im.mappings.pixels.dtype == torch.int16
    assert torch.equal(im[torch.tensor([1])].rollings, torch.tensor([15]))
    assert torch.equal(im.clone().rollings, im.rollings)
    from deepviewagg_b200.core.multimodal.image import SameSettingImageBatch
    assert torch.equal(SameSettingImageBatch.from_data_list([im, im]).rollings, torch.tensor([3, 15, 3, 15]))
    assert im.settings_hash == _tiny().settings_hash
    with pytest.raises(AssertionError):
        im.clone().update_cropping((8, 8), torch.zeros(2, 2, dtype=torch.long)).update_rollings(torch.zeros(2).long())


def test_update_cropping_accumulates_offsets():
    im = _tiny()
    im.update_cropping((8, 4), torch.tensor([[2, 1], [8, 4]]))
    assert im.crop_size == (8, 4) and torch.equal(im.crop_offsets, torch.tensor([[2, 1], [8, 4]]))
    assert torch.equal(im.x[1], _tiny().x[1, :, 4:8, 8:16])
    im.update_cropping((4, 2), torch.tensor([[1, 1], [0, 2]]))
    assert torch.equal(im.crop_offsets, torch.tensor([[3, 2], [8, 6]]))
    assert torch.equal(im.x[0], _tiny().x[0, :, 2:4, 3:7])


def test_entry_points_reject_bad_arguments():
    lib = _lib.load()
    n0 = _lib.launch_count()
    assert lib.dva_mapping_image_stats(None, None, None, 0, -1, 4, 0, None, None, None, None) == _lib.DVA_EINVAL
    assert lib.dva_mapping_image_stats(None, None, None, 3, 4, 4, 0, None, None, None, None) == _lib.DVA_EUNSUPPORTED
    assert lib.dva_mapping_image_stats(None, None, None, 0, 4, 4, 8, None, None, None, None) == _lib.DVA_EINVAL
    assert b"mapping_image_stats" in lib.dva_last_error()
    for ar in (0, 257):
        assert lib.dva_center_roll(None, 4, ar, 256, None, None) == _lib.DVA_EINVAL
    assert lib.dva_center_roll(None, 4, 16, 0, None, None) == _lib.DVA_EINVAL
    assert lib.dva_image_remap(None, None, 2, 3, 8, 8, 8, 8, 8, 0, None, None, 0, None) == _lib.DVA_EUNSUPPORTED
    assert lib.dva_image_remap(None, None, 2, 3, 8, 8, 9, 8, 1, 0, None, None, 0, None) == _lib.DVA_EINVAL
    assert lib.dva_image_remap(None, None, 2, 3, 8, 8, 8, 8, 1, 0, None, None, 0, None) == _lib.DVA_EINVAL
    assert lib.dva_coverage_index_workspace_bytes(100, 4, 50) > 0
    assert lib.dva_coverage_index(None, None, 100, 4, 50, None, None, None, 0, None) == _lib.DVA_EINVAL
    ws = lib.dva_coverage_index_workspace_bytes(100, 4, 50)
    assert lib.dva_coverage_pick(4, 100, 4, 50, None, None, None, ws, None) == _lib.DVA_EINVAL
    assert lib.dva_coverage_pick(-1, 100, 4, 50, None, None, None, ws, None) == _lib.DVA_EINVAL
    assert b"coverage_pick" in lib.dva_last_error()
    assert _lib.launch_count() == n0
