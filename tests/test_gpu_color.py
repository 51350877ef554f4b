"""Colour transforms on CUDA containers (csrc/image_color.cu): equal to the CPU path bit for bit on every fixture
in both memory formats and for 0, 1 and 3 images; a full-size sample through the four transforms without a host
synchronisation; the S3DIS train chain on CUDA against the CPU chain, then one UnimodalBranch step."""
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
from oracle import color_oracle as O
from test_color import check_float, check_jitter_equals_oracle, container, jitter_cases, jitter_fixture, run_jitter

sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_transforms import chain, synthetic_sample  # noqa: E402

pytestmark = pytest.mark.gpu

FORMATS = [torch.contiguous_format, torch.channels_last]


@pytest.mark.parametrize("memory_format", FORMATS)
def test_jitter_cuda_equals_oracle(memory_format):
    check_jitter_equals_oracle("cuda", memory_format)


@pytest.mark.parametrize("memory_format", FORMATS)
@pytest.mark.parametrize("n_img", [0, 1, 3])
def test_jitter_cuda_equals_cpu(memory_format, n_img):
    z = jitter_fixture()
    for case in jitter_cases(z):
        cpu = run_jitter(z, case, "cpu", memory_format, n_img=n_img)
        gpu = run_jitter(z, case, "cuda", memory_format, n_img=n_img)
        for a, b in zip(cpu, gpu):
            assert b.x.is_cuda and b.x.is_contiguous(memory_format=memory_format)
            assert torch.equal(a.x, b.x.cpu()), (case, n_img)


def test_jitter_cuda_consumes_the_same_draws():
    z = jitter_fixture()
    for case in ("two_settings", "s3dis_0"):
        after = {}
        for device in ("cpu", "cuda"):
            run_jitter(z, case, device, n_img=0)
            after[device] = torch.rand(1)
        assert torch.equal(after["cpu"], after["cuda"])


@pytest.mark.parametrize("memory_format", FORMATS)
def test_to_float_and_normalize_cuda_equal_fixtures(memory_format):
    check_float("cuda", memory_format)


@pytest.mark.parametrize("memory_format", FORMATS)
def test_to_float_and_normalize_cuda_equal_cpu_odd_shapes(memory_format):
    for shape in [(3, 3, 61, 97), (2, 3, 16, 16), (1, 1, 7, 5), (2, 4, 9, 33), (0, 3, 4, 4)]:
        g = torch.Generator().manual_seed(sum(shape))
        x = torch.randint(0, 256, shape, dtype=torch.uint8, generator=g).contiguous(memory_format=memory_format)
        mean, std = [0.1, 0.2, 0.3, 0.4][:shape[1]], [0.3, 0.25, 0.5, 0.7][:shape[1]]
        outs = {}
        for device in ("cpu", "cuda"):
            im = container(x.numpy(), device, memory_format)
            _, im = T.ToFloatImage()(None, im)
            f = im.x
            _, im = T.Normalize(mean, std)(None, im)
            outs[device] = (f, im.x)
        for a, b in zip(outs["cpu"], outs["cuda"]):
            assert b.numel() == 0 or b.is_contiguous(memory_format=memory_format), shape
            assert torch.equal(a, b.cpu()), shape
    # the kernels reject what they do not run, without a launch
    with pytest.raises(TypeError):
        ops.image_to_float(torch.zeros(1, 5, 4, 4, device="cuda"))
    with pytest.raises(TypeError):
        ops.color_jitter_u8(torch.zeros(1, 3, 4, 4, device="cuda"), [("brightness", 1.2)])
    with pytest.raises(TypeError):
        T.Normalize()(None, container(np.zeros((1, 3, 4, 4), np.float64), "cuda"))


def test_full_size_sample_without_sync():
    x = torch.from_numpy(O.color_input("formula", 4, 512, 1024)).cuda().contiguous(memory_format=torch.channels_last)
    im = container(x.cpu().numpy(), "cuda", torch.channels_last)
    torch.cuda.synchronize()
    chain_ = [T.ToImageData(), T.ColorJitter(0.6, 0.6, 0.7), T.ToFloatImage(), T.Normalize()]
    torch.manual_seed(0)
    torch.cuda.set_sync_debug_mode("error")
    try:
        for t in chain_:
            _, im = t(None, im)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert isinstance(im, ImageData) and im[0].x.dtype == torch.float32
    assert im[0].x.is_contiguous(memory_format=torch.channels_last)
    ref = container(x.cpu().numpy(), "cpu", torch.channels_last)
    torch.manual_seed(0)
    for t in chain_:
        _, ref = t(None, ref)
    assert torch.equal(ref[0].x, im[0].x.cpu())


def test_s3dis_train_chain_cuda_equals_cpu_then_branch_step():
    from deepviewagg_b200.modules.multimodal.fusion import BimodalFusion
    from deepviewagg_b200.modules.multimodal.modules import UnimodalBranch
    from deepviewagg_b200.modules.multimodal.pooling import BimodalCSRPool
    data, images = synthetic_sample(seed=3, n_points=50_000, n_img=24)
    steps = [t for name, t in chain() if name != "RandomHorizontalFlip"]
    steps += [T.ColorJitter(0.6, 0.6, 0.7), T.RandomHorizontalFlip(p=0.5), T.ToFloatImage(), T.Normalize()]
    results = {}
    for device in ("cpu", "cuda"):
        d = types.SimpleNamespace(pos=data.pos.to(device), mapping_index=data.mapping_index.to(device))
        im = images.clone().to(device)
        torch.manual_seed(5)
        np.random.seed(5)
        for t in steps:
            d, im = t(d, im)
        results[device] = (d, im)
    cpu, gpu = results["cpu"][1], results["cuda"][1]
    assert isinstance(gpu, ImageData) and len(list(cpu)) == len(list(gpu)) >= 2
    for a, b in zip(cpu, gpu):
        assert b.x.dtype == torch.float32 and torch.equal(a.x, b.x.cpu())
        assert torch.equal(a.mappings.pixels, b.mappings.pixels.cpu())
    d, mod = results["cuda"]
    xs = []
    for im in mod:
        im._x = im.x.contiguous(memory_format=torch.channels_last).requires_grad_(True)
        xs.append(im._x)
    n = d.pos.shape[0]
    branch = UnimodalBranch(None, BimodalCSRPool("max"), BimodalCSRPool("mean"), BimodalFusion("concatenation"),
                            out_channels=6).cuda()
    x_3d = torch.randn(n, 3, device="cuda", requires_grad=True)
    out = branch({"x_3d": x_3d, "x_seen": None, "modalities": {"image": mod}}, "image")
    assert out["x_3d"].shape[0] == n and torch.isfinite(out["x_3d"]).all()
    grads = torch.autograd.grad(out["x_3d"].square().sum(), [x_3d] + xs)
    assert all(torch.isfinite(gr).all() for gr in grads)
    assert any(float(gr.abs().sum()) > 0 for gr in grads[1:])
