"""Colour transforms (ColorJitter, ToFloatImage, Normalize, ToImageData) on CPU containers against the fixtures
executed on the reference with torchvision (tests/golden/color_{jitter,float}.npz), through the numpy oracle
(oracle/color_oracle.py).  The check_* helpers take a device and a memory format and are shared with
tests/test_gpu_color.py."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from deepviewagg_b200 import _lib
from deepviewagg_b200.core.multimodal import transforms as T
from deepviewagg_b200.core.multimodal.image import ImageData, SameSettingImageData
from oracle import color_oracle as O


def jitter_fixture():
    return np.load(os.path.join(GOLDEN, "color_jitter.npz"), allow_pickle=False)


def float_fixture():
    return np.load(os.path.join(GOLDEN, "color_float.npz"), allow_pickle=False)


def jitter_cases(z):
    return sorted({k.split("/")[1] for k in z.files if k.startswith("jitter/")})


def settings(z, case):
    """[(prefix, input x)] of a case, the input checked against its stored shape and sum"""
    out = []
    for s in range(int(z[f"jitter/{case}/n_settings"])):
        p = f"jitter/{case}/{s}/"
        B, _, H, W = z[p + "shape"].tolist()
        x = O.color_input(str(z[p + "kind"]), B, H, W)
        assert int(x.astype(np.int64).sum()) == int(z[p + "input_sum"]), p
        out.append((p, x))
    return out


def factors(z, p):
    return tuple(None if np.isnan(v) else float(v) for v in z[p + "factors"])


def container(x, device, memory_format=torch.contiguous_format):
    t = torch.from_numpy(np.ascontiguousarray(x)).to(device).contiguous(memory_format=memory_format)
    return SameSettingImageData(pos=torch.zeros(x.shape[0], 3, device=device), ref_size=(x.shape[3], x.shape[2]), x=t)


def run_jitter(z, case, device, memory_format=torch.contiguous_format, n_img=None):
    """the package's ColorJitter on a case under its seed; n_img keeps the first n images of every setting"""
    ims = [container(x[:n_img], device, memory_format) for _, x in settings(z, case)]
    images = ims[0] if len(ims) == 1 else ImageData(ims)
    torch.manual_seed(int(z[f"jitter/{case}/seed"]))
    _, out = T.ColorJitter(*z[f"jitter/{case}/config"].tolist())(None, images)
    return [out] if len(ims) == 1 else list(out)


def _out_matches(z, p, y):
    if p + "out" in z.files:
        return np.array_equal(y, z[p + "out"])
    return hashlib.sha256(np.ascontiguousarray(y).tobytes()).hexdigest() == str(z[p + "out_sha256"])


def test_oracle_with_torch_mean_equals_fixtures():
    z = jitter_fixture()
    cases = jitter_cases(z)
    assert len(cases) >= 17
    for case in cases:
        for p, x in settings(z, case):
            means = z[p + "torch_mean"] if p + "torch_mean" in z.files else None
            y, steps = O.color_jitter(x, z[p + "fn_idx"], factors(z, p), means)
            assert _out_matches(z, p, y), p
            if means is not None:
                assert np.array_equal(steps[0][0], means)
                assert np.array_equal(O.exact_mean(O.grayscale(steps[0][1])), z[p + "exact_mean"]), p


def test_fixtures_cover_every_order_and_an_inexact_torch_mean():
    z = jitter_fixture()
    for tag in ("s3dis", "kitti"):
        orders = {tuple(int(i) for i in z[f"jitter/{c}/0/fn_idx"] if i < 3) for c in jitter_cases(z)
                  if c.startswith(tag + "_")}
        assert len(orders) == 6, tag
    # the large case: torch's fp32 mean is an ulp away from the exact one
    assert not np.array_equal(z["jitter/large/0/torch_mean"], z["jitter/large/0/exact_mean"])


def test_draws_equal_recorded():
    z = jitter_fixture()
    for case in jitter_cases(z):
        torch.manual_seed(int(z[f"jitter/{case}/seed"]))
        cj = T.ColorJitter(*z[f"jitter/{case}/config"].tolist())
        for p, _ in settings(z, case):
            fn_idx, seq = cj.get_params()
            assert np.array_equal(fn_idx.numpy(), z[p + "fn_idx"]), p
            f = factors(z, p)
            names = ("brightness", "contrast", "saturation")
            assert seq == [(names[i], f[i]) for i in z[p + "fn_idx"].tolist() if i < 3 and f[i] is not None], p


def check_jitter_equals_oracle(device, memory_format):
    """the package's ColorJitter (exact mean) equals the oracle with the exact mean, for every case"""
    z = jitter_fixture()
    for case in jitter_cases(z):
        outs = run_jitter(z, case, device, memory_format)
        for (p, x), im in zip(settings(z, case), outs):
            y, _ = O.color_jitter(x, z[p + "fn_idx"], factors(z, p), None)
            assert im.x.device.type == torch.device(device).type and im.x.dtype == torch.uint8
            assert im.x.is_contiguous(memory_format=memory_format), p
            assert np.array_equal(im.x.cpu().numpy(), y), p


@pytest.mark.parametrize("memory_format", [torch.contiguous_format, torch.channels_last])
def test_cpu_jitter_equals_oracle_exact_mean(memory_format):
    check_jitter_equals_oracle("cpu", memory_format)


def test_cpu_jitter_differs_from_reference_only_near_integers():
    """exact mean vs torch's mean: a pixel may differ by 1 only where the contrast blend lies within the mean
    shift of an integer (the oracle flags those); the count is printed"""
    z = jitter_fixture()
    flagged_total, differing = 0, 0
    for case in jitter_cases(z):
        outs = run_jitter(z, case, "cpu")
        for (p, x), im in zip(settings(z, case), outs):
            got = im.x.numpy()
            if p + "torch_mean" not in z.files:
                assert _out_matches(z, p, got), p
                continue
            ref, steps = O.color_jitter(x, z[p + "fn_idx"], factors(z, p), z[p + "torch_mean"])
            assert _out_matches(z, p, ref), p
            flag = O.contrast_near_integer(steps[0][1], factors(z, p)[1], z[p + "torch_mean"], z[p + "exact_mean"])
            flag_px = flag.any(axis=1, keepdims=True)
            d = got.astype(np.int16) - ref.astype(np.int16)
            flagged_total += int(flag_px.sum())
            differing += int((d != 0).any(axis=1).sum())
            assert not ((d != 0) & ~flag_px).any(), p
            assert np.abs(d).max(initial=0) <= 1, p
    print(f"pixels within the mean shift of an integer: {flagged_total}; differing from the reference: {differing}")


def check_float(device, memory_format):
    z = float_fixture()
    x = O.color_input(str(z["float/kind"]), *z["float/shape"].tolist()[:1], *z["float/shape"].tolist()[2:])
    assert int(x.astype(np.int64).sum()) == int(z["float/input_sum"])
    im = container(x, device, memory_format)
    _, im = T.ToFloatImage()(None, im)
    assert im.x.dtype == torch.float32 and im.x.is_contiguous(memory_format=memory_format)
    assert np.array_equal(im.x.cpu().numpy(), z["float/to_float"])
    _, im = T.Normalize()(None, im)
    assert im.x.is_contiguous(memory_format=memory_format)
    assert np.array_equal(im.x.cpu().numpy(), z["float/normalize"])
    im = container(x, device, memory_format)
    _, im = T.ToFloatImage()(None, im)
    _, im = T.Normalize(mean=z["float/custom_mean"].tolist(), std=z["float/custom_std"].tolist())(None, im)
    assert np.array_equal(im.x.cpu().numpy(), z["float/normalize_custom"])


@pytest.mark.parametrize("memory_format", [torch.contiguous_format, torch.channels_last])
def test_cpu_to_float_and_normalize_equal_fixtures(memory_format):
    check_float("cpu", memory_format)


def test_oracle_float_equals_fixtures():
    z = float_fixture()
    x = O.color_input(str(z["float/kind"]), 3, *z["float/shape"].tolist()[2:])
    f = O.to_float(x)
    assert np.array_equal(f, z["float/to_float"])
    assert np.array_equal(O.normalize(f, [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]), z["float/normalize"])
    assert np.array_equal(O.normalize(f, z["float/custom_mean"], z["float/custom_std"]), z["float/normalize_custom"])


def test_to_image_data():
    z = float_fixture()
    assert int(z["to_image_data/n_settings"]) == 1 and bool(z["to_image_data/x_equal"])
    im = container(O.color_input("formula", 2, 5, 7), "cpu")
    _, out = T.ToImageData()(None, im)
    assert isinstance(out, ImageData) and out.num_settings == 1 and out[0] is im
    _, again = T.ToImageData()(None, out)
    assert isinstance(again, ImageData) and again.num_settings == 1 and again[0] is im


def test_argument_errors():
    im = container(O.color_input("formula", 2, 5, 7), "cpu")
    im.x = im.x.float()
    with pytest.raises(TypeError):
        T.ColorJitter(0.5, 0.5, 0.5)(None, im)
    with pytest.raises(TypeError):
        T.ColorJitter(0.5)(None, container(np.zeros((2, 4, 5, 7), np.uint8), "cpu"))
    with pytest.raises(ValueError):
        T.ColorJitter(brightness=-1)
    with pytest.raises(TypeError):
        T.Normalize()(None, container(O.color_input("formula", 2, 5, 7), "cpu"))
    with pytest.raises(ValueError):
        T.Normalize(std=[1.0, 0.0, 1.0])(None, im)
    # empty settings consume their draw and stay as they are
    empty = container(np.zeros((0, 3, 5, 7), np.uint8), "cpu")
    torch.manual_seed(0)
    _, out = T.ColorJitter(0.5, 0.5, 0.5)(None, empty)
    after = torch.rand(1)
    torch.manual_seed(0)
    T.ColorJitter(0.5, 0.5, 0.5).get_params()
    assert out.x.shape == (0, 3, 5, 7) and torch.equal(after, torch.rand(1))


def test_entry_points_reject_bad_arguments_without_launch():
    lib = _lib.load()
    n0 = _lib.launch_count()
    assert lib.dva_color_jitter_u8_workspace_bytes(5) == 40
    j = lambda *a: lib.dva_color_jitter_u8(None, None, *a)  # noqa: E731
    assert j(-1, 4, 4, 0, 1, 0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, None, 0, None) == _lib.DVA_EINVAL       # negative B
    assert j(1, 4, 4, 0, 4, 0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, None, 0, None) == _lib.DVA_EINVAL        # 4 ops
    assert j(1, 4, 4, 0, 1, 3, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, None, 0, None) == _lib.DVA_EINVAL        # hue code
    assert j(1, 4, 4, 0, 2, 0x00, 1.0, 0.0, 1.0, 0.0, 0.0, 0.0, None, 0, None) == _lib.DVA_EINVAL     # op twice
    assert j(1, 4, 4, 0, 1, 0, -1.0, 2.0, 0.0, 0.0, 0.0, 0.0, None, 0, None) == _lib.DVA_EINVAL       # negative factor
    assert j(2, 4, 4, 0, 1, 1, 1.5, -0.5, 0.0, 0.0, 0.0, 0.0, None, 0, None) == _lib.DVA_EINVAL       # no workspace
    assert b"workspace" in lib.dva_last_error()
    assert j(1, 4, 4, 0, 1, 0, 1.5, -0.5, 0.0, 0.0, 0.0, 0.0, None, 0, None) == _lib.DVA_EINVAL       # null images
    assert j(0, 4, 4, 0, 1, 0, 1.5, -0.5, 0.0, 0.0, 0.0, 0.0, None, 0, None) == 0                     # B = 0: no-op
    f = lambda *a: lib.dva_image_to_float(None, 1, None, *a, 0, *([0.0] * 4), *([1.0] * 4), None)  # noqa: E731
    assert f(1, 5, 4, 4) == _lib.DVA_EUNSUPPORTED
    assert f(1, 0, 4, 4) == _lib.DVA_EUNSUPPORTED
    assert f(-1, 3, 4, 4) == _lib.DVA_EINVAL
    assert f(1, 3, 4, 4) == _lib.DVA_EINVAL                                                        # null pointers
    assert f(0, 3, 4, 4) == 0
    assert _lib.launch_count() == n0


def test_package_does_not_import_torchvision():
    code = ("import sys; import deepviewagg_b200.core.multimodal.transforms, deepviewagg_b200.ops; "
            "assert 'torchvision' not in sys.modules, 'torchvision imported'")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]


def test_against_torchvision_when_installed():
    """direct check of the CPU path against torchvision.transforms.ColorJitter on random images: equal wherever
    the contrast mean is not involved, and at most 1 apart otherwise"""
    tv = pytest.importorskip("torchvision.transforms")
    g = np.random.default_rng(0)
    for trial in range(12):
        cfg = [(0.6, 0.6, 0.7), (0.2, 0.2, 0.2), (0.0, 0.0, 0.5), (0.5, 0.0, 0.0)][trial % 4]
        x = torch.from_numpy(g.integers(0, 256, (2, 3, 33, 47), dtype=np.uint8))
        torch.manual_seed(trial)
        ref = tv.ColorJitter(*cfg)(x)
        torch.manual_seed(trial)
        _, im = T.ColorJitter(*cfg)(None, container(x.numpy(), "cpu"))
        d = (im.x.int() - ref.int()).abs()
        assert int(d.max()) <= (1 if cfg[1] else 0), trial
        ref_n = tv.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])(im.x.float() / 255)
        assert torch.equal(T.Normalize()(None, T.ToFloatImage()(None, im)[1])[1].x, ref_n)
