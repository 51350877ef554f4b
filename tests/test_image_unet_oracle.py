"""The image UNet on the CPU: the float64 oracle (oracle/image_unet_oracle.py) against the fixtures made by
executing the reference's UNet (oracle/make_golden_image_unet.py); standardize_weights on transposed weights; every
shipped UNet config built with the reference's state-dict keys and shapes; the options and sizes that raise; and
fetch_arguments_from_list against the reference's own."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from deepviewagg_b200.modules.multimodal.modalities import image as I
from oracle import image_unet_oracle as O
from oracle import ref_loader

DOWN = [(3, 1, 1)] + [(2, 2, 0)] * 4
UP = {"unet5": [(2, 2, 0)] * 4 + [(3, 1, 1)], "unet4": [(2, 2, 0)] * 4}
CASES = ["unet5_b2", "unet4_b1"]


def fixture(name):
    return np.load(os.path.join(GOLDEN, f"image_unet_{name}.npz"), allow_pickle=False)


def unpack(z):
    """(keys, parameters, gradients, float64 gradient norms) of a fixture, each a dict over the state-dict keys; the
    parameters are float32-exact, the gradients the float64 reference's rounded to float32."""
    keys = [str(k) for k in z["keys"]]
    shapes = [json.loads(str(s)) for s in z["shapes"]]
    offs = np.cumsum([0] + [int(np.prod(s)) for s in shapes])

    def cut(a):
        return {k: torch.from_numpy(a[o:e].reshape(s)) for k, o, e, s in zip(keys, offs[:-1], offs[1:], shapes)}
    return keys, cut(z["params"]), cut(z["grads"]), dict(zip(keys, (float(n) for n in z["grad_norms"])))


def configs():
    z = np.load(os.path.join(GOLDEN, "image_unet_configs.npz"), allow_pickle=False)
    return z, [(str(n), json.loads(str(z[f"opt{i}"])), str(z[f"norm{i}"])) for i, n in enumerate(z["names"])]


def small_opt(topo, f=4):
    """The fixture topologies (oracle/make_golden_image_unet.py) as a plain dict."""
    down = dict(module_name="ResNetDown", block="ResBlock", normalization="GroupNorm", weight_standardization=True,
                N=[0, 2, 2, 2, 2], stride=[1, 2, 2, 2, 2], kernel_size=[3, 2, 2, 2, 2], padding=[1, 0, 0, 0, 0],
                down_conv_nn=[[4, f], [f, f], [f, 2 * f], [2 * f, 4 * f], [4 * f, 8 * f]])
    nn_up = [[8 * f, 4 * f, 4 * f], [4 * f, 2 * f, 3 * f], [3 * f, f, 2 * f], [2 * f, f, f]]
    shapes = UP[topo]
    if topo == "unet5":
        nn_up.append([f, 0, f])
    up = dict(module_name="ResNetUp", block="ResBlock", normalization="GroupNorm", weight_standardization=True, N=1,
              kernel_size=[s[0] for s in shapes], stride=[s[1] for s in shapes], padding=[s[2] for s in shapes],
              up_conv_nn=nn_up)
    return dict(down_conv=down, up_conv=up, last_conv=dict(input_nc=f, output_nc=13))


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_fixtures(name):
    """The fixture stores the reference's results rounded to float32 (at most 2^-24 relative per element) and their
    float64 norms: the oracle matches the first to float32 rounding and the second to 1e-12."""
    z = fixture(name)
    keys, params, grads, norms = unpack(z)
    sd = {k: params[k].double().requires_grad_(True) for k in keys}
    x = torch.from_numpy(z["x"]).double().requires_grad_(True)
    y = O.unet(x, sd, DOWN, UP[name.split("_")[0]], last={})
    yd = y.detach()
    assert float((yd - torch.from_numpy(z["y"]).double()).abs().max() / yd.abs().max()) <= 2.0 ** -23
    assert abs(float(yd.norm()) - float(z["norm_y"])) <= 1e-12 * float(z["norm_y"])
    g = torch.autograd.grad(y, [x] + list(sd.values()), torch.from_numpy(z["gy"]).double())
    assert float((g[0] - torch.from_numpy(z["gx"]).double()).norm() / g[0].norm()) <= 2.0 ** -23
    assert abs(float(g[0].norm()) - float(z["norm_gx"])) <= 1e-12 * float(z["norm_gx"])
    for k, gk in zip(keys, g[1:]):
        ref = grads[k].double()
        assert float((gk - ref).norm()) <= 2.0 ** -23 * max(float(gk.norm()), 1e-30), k
        assert abs(float(gk.norm()) - norms[k]) <= 1e-10 * max(norms[k], 1e-30), k


@pytest.mark.parametrize("name", CASES)
def test_fixture_state_dict_loads_strictly(name):
    z = fixture(name)
    net = I.UNet(small_opt(name.split("_")[0]))
    keys, params, _, _ = unpack(z)
    assert list(net.state_dict().keys()) == keys
    assert all(tuple(params[k].shape) == tuple(v.shape) for k, v in net.state_dict().items())
    net.load_state_dict(params, strict=True)


def test_standardize_weights_on_transposed_weights_equals_executed_reference():
    z, _ = configs()
    tags = sorted({k[:-2] for k in z.files if k.startswith("ws_") and k.endswith("_w")})
    assert len(tags) == 4
    for t in tags:
        w = torch.from_numpy(z[t + "_w"])
        ref = torch.from_numpy(z[t + "_ref"])
        tol = 1e-6 if w.dtype == torch.float32 else 1e-13
        got = I.standardize_weights(w)
        assert got.dtype == w.dtype and torch.allclose(got, ref, rtol=tol, atol=tol), t
        assert torch.allclose(O.E.standardize(w.double()), ref.double(), rtol=10 * tol, atol=10 * tol), t


class AttrDict(dict):
    """A stand-in for omegaconf's DictConfig: a dict with attribute access."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


def attr(o):
    if isinstance(o, dict):
        return AttrDict({k: attr(v) for k, v in o.items()})
    if isinstance(o, list):
        return [attr(v) for v in o]
    return o


def test_every_shipped_unet_config_has_the_reference_state_dict():
    z, cfgs = configs()
    assert len(cfgs) == 16
    n_gn = 0
    for i, (name, opt, norm) in enumerate(cfgs):
        if norm != "GroupNorm":
            with pytest.raises(NotImplementedError, match="normalization"):
                I.UNet(opt)
            continue
        n_gn += 1
        for o in (opt, attr(opt)):
            sd = I.UNet(o).state_dict()
            assert list(sd.keys()) == [str(k) for k in z[f"keys{i}"]], name
            assert [json.dumps(list(v.shape)) for v in sd.values()] == [str(s) for s in z[f"shapes{i}"]], name
    assert n_gn == 15


def test_reference_behaviour_recorded_by_the_fixtures():
    """The reference cannot run persistent dropout in last_conv (UNet.forward passes no reset) nor, on current torch,
    ConvTranspose2dWS.forward (_output_padding lacks num_spatial_dims); ours pass reset and do not call it."""
    z, _ = configs()
    assert "reset" in str(z["persistent_drop_error"]) and str(z["persistent_drop_error"]).startswith("TypeError")
    assert "num_spatial_dims" in str(z["convt_error"])
    net = I.UNet(small_opt("unet4") | {"last_conv": dict(input_nc=4, output_nc=13, in_drop=0.5,
                                                         persistent_drop=True)})
    assert isinstance(net.last.input_dropout, I.PersistentDropout2d)


@pytest.mark.parametrize("kw, word", [
    (dict(normalization="BatchNorm2d"), "normalization"),
    (dict(weight_standardization=False), "weight_standardization"),
    (dict(block="BottleneckBlock"), "block"),
    (dict(padding_mode="reflect"), "padding_mode"),
    (dict(dilation=2), "dilation"),
    (dict(kernel_size=4), "kernel_size"),
    (dict(N=-1), "N="),
])
def test_resnet_up_unsupported_options_raise(kw, word):
    base = dict(up_conv_nn=[8, 4, 4], kernel_size=2, stride=2, padding=0, N=1, block="ResBlock",
                normalization="GroupNorm", weight_standardization=True)
    with pytest.raises(NotImplementedError, match=word):
        I.ResNetUp(**{**base, **kw})


def test_unary_conv_and_unet_unsupported_options_raise():
    with pytest.raises(NotImplementedError, match="normalization"):
        I.UnaryConv(4, 13, normalization="GroupNorm")
    with pytest.raises(NotImplementedError, match="activation"):
        I.UnaryConv(4, 13, activation="LeakyReLU")
    with pytest.raises(NotImplementedError, match="innermost"):
        I.UNet(small_opt("unet4") | {"innermost": dict(module_name="BottleneckBlock")})
    with pytest.raises(NotImplementedError, match="compact"):
        I.UNet(dict(down_conv=[small_opt("unet4")["down_conv"]], up_conv=small_opt("unet4")["up_conv"]))
    with pytest.raises(NotImplementedError, match="ConvTranspose2dWS"):
        I.ConvTranspose2dWS(4, 8, 2, stride=2)(torch.zeros(1, 4, 2, 2))


def test_module_tree_of_the_decoder():
    up = I.ResNetUp(up_conv_nn=[256, 128, 128], kernel_size=2, stride=2, padding=0, N=1, block="ResBlock",
                    normalization="GroupNorm", weight_standardization=True, module_name="ResNetUp")
    conv, norm, act = up.conv_in
    assert isinstance(conv, I.ConvTranspose2dWS) and conv.weight.shape == (256, 256, 2, 2)
    assert norm.num_groups == 16 and isinstance(act, I.ReLUWS)
    blk = up.blocks[0]
    assert blk.block[0].weight.shape == (384, 128, 3, 3) and blk.block[0].padding_mode == "zeros"
    assert type(blk.downsample[0]) is torch.nn.Conv2d and blk.downsample[0].bias is not None
    last = I.UnaryConv(32, 13, weight_standardization=True, activation="ReLU", in_drop=0.5)
    assert isinstance(last.conv, I.Conv2dWS) and last.activation is I.ReLUWS
    assert isinstance(last.input_dropout, I.Dropout2d) and last.output_dropout is None
    assert I.ResNetUp(up_conv_nn=[]).conv_in is None


def test_bad_sizes_raise_value_error_naming_the_stage():
    net = I.UNet(small_opt("unet5"))
    assert net.check_sizes(48, 32) == (48, 32)
    with pytest.raises(ValueError, match=r"UNet up stage 2: the skip connection is 25x16 but the map it joins is "
                                         r"24x16"):
        net.check_sizes(50, 32)
    with pytest.raises(ValueError, match=r"UNet up stage 2: the skip connection is 24x17 but the map it joins is "
                                         r"24x16"):
        net.check_sizes(48, 34)


def test_fetch_arguments_from_list_restatement():
    opt = dict(module_name="ResNetUp", N=1, kernel_size=[2, "1+2"], up_conv_nn=[[8, 4, 4], [4, 0, 4]],
               block_names=["a", "b"], empty=[])
    assert I.fetch_arguments_from_list(opt, 1, I.SPECIAL_NAMES) == dict(
        module_name="ResNetUp", N=1, kernel_size=3, up_conv_nn=[4, 0, 4], block_names="b", empty=[])


@pytest.mark.needs_reference
@pytest.mark.skipif(not ref_loader.available(), reason="reference not available")
def test_fetch_arguments_from_list_equals_the_reference():
    from oracle import make_golden_image_unet as MU
    cfg = MU.load_reference_config()
    _, cfgs = configs()
    for _, opt, _ in cfgs:
        for part in ("down_conv", "up_conv", "last_conv"):
            sub = opt.get(part)
            if sub is None:
                continue
            n = max([len(v) for v in sub.values() if isinstance(v, list)] + [1])
            for i in range(n):
                ref = cfg.fetch_arguments_from_list(MU.to_cfg(sub), i, I.SPECIAL_NAMES)
                assert I.fetch_arguments_from_list(sub, i, I.SPECIAL_NAMES) == ref
                assert I.fetch_arguments_from_list(attr(sub), i, I.SPECIAL_NAMES) == ref
