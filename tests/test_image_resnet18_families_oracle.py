"""The ImageNet and Cityscapes ResNet-18 encoders without a GPU: the float64 restatement
oracle/image_resnet18_families_oracle.py against the fixtures made by executing the reference's wrappers
(oracle/make_golden_image_resnet18_families.py), the classes' state-dict keys against the reference's, both
checkpoint loaders, the frozen / train() semantics, the BatchNorm bookkeeping and the new C ABI entries' argument
errors."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from deepviewagg_b200 import _lib, ops
from deepviewagg_b200.modules.multimodal.modalities import image as I
from oracle import image_resnet18_families_oracle as O

_LAYERS = ["Layer0", "Layer1", "Layer2", "Layer3", "Layer4"]
CLASSES = ([f"ResNet18Truncated{n}" for n in _LAYERS] + [f"ResNet18{n}" for n in _LAYERS] + ["ResNet18Pyramid"]
           + [f"CityscapesResNet18Truncated{n}" for n in _LAYERS] + [f"CityscapesResNet18{n}" for n in _LAYERS]
           + ["CityscapesResNet18Pyramid", "CityscapesResNet18"])
CASES = {  # oracle/make_golden_image_resnet18_families.py:CASES
    "rn_tl4_train": ("ResNet18TruncatedLayer4", {}, True, (2, 3, 61, 45), 11),
    "rn_layer2_eval": ("ResNet18Layer2", {}, False, (1, 64, 15, 18), 12),
    "rn_pyramid_train": ("ResNet18Pyramid", {"scale_factor": -1}, True, (2, 3, 8, 10), 13),
    "cs_tl4_train": ("CityscapesResNet18TruncatedLayer4", {}, True, (2, 3, 60, 44), 14),
    "cs_layer1_train": ("CityscapesResNet18Layer1", {}, True, (2, 128, 9, 11), 15),
    "cs_full_train": ("CityscapesResNet18", {}, True, (2, 3, 50, 66), 16),
    "cs_pyramid_eval": ("CityscapesResNet18Pyramid", {}, False, (2, 3, 10, 8), 17),
}
LAYER0 = {"imagenet": ("ResNet18TruncatedLayer0", (2, 3, 50, 66), 21),
          "cityscapes": ("CityscapesResNet18TruncatedLayer0", (2, 3, 52, 66), 22)}


def family(m):
    return "cityscapes" if type(m).__name__.startswith("Cityscapes") else "imagenet"


def oracle_args(m):
    """(family, layers, prefixes) of module m for O.forward."""
    if isinstance(m, I.CityscapesResNet18):
        return "cityscapes", list(I._TRUNK_LAYERS), list(I._TRUNK_LAYERS)
    return family(m), list(m._LAYERS), None


def run_oracle(m, state, x, seed, pyramid):
    """The oracle's step of m on (state, x): y, grads of (x, params), the state after the step, parameter names."""
    fam, layers, prefixes = oracle_args(m)
    p = {k: v.clone() for k, v in state.items()}
    names = [k for k, _ in m.named_parameters()]
    for k in names:
        p[k].requires_grad_(True)
    x = x.clone().requires_grad_(True)
    y = O.forward(x, p, fam, layers, m.training, m.scale_factor, pyramid, prefixes=prefixes)
    gy = torch.from_numpy(O.hash_grid(seed, 60000, tuple(y.shape), 8, 3))
    return y, torch.autograd.grad(y, [x] + [p[k] for k in names], gy), p, names


def check_step(g, y, grads, p, names, seed, prefix=""):
    u = 2.0 ** -24
    assert np.abs(y.detach().float().numpy() - g[prefix + "y"]).max() <= u * np.abs(g[prefix + "y"]).max()
    assert np.abs(grads[0].float().numpy() - g[prefix + "gx"]).max() <= u * np.abs(g[prefix + "gx"]).max()
    assert abs(float(y.detach().norm()) / float(g[prefix + "y_norm"]) - 1) <= 1e-12
    assert abs(float(grads[0].norm()) / float(g[prefix + "gx_norm"]) - 1) <= 1e-12
    for tag, (k, gp) in enumerate(zip(names, grads[1:])):
        assert abs(float(gp.norm()) / float(g[f"{prefix}gnorm:{k}"]) - 1) <= 1e-12, k
        proj = float((gp * O.projection(seed, tag, tuple(gp.shape))).sum())
        assert abs(proj - float(g[f"{prefix}gproj:{k}"])) <= 1e-12 * float(g[f"{prefix}gnorm:{k}"]) * gp.numel() ** .5
    for k in p:
        if k.endswith((".running_mean", ".running_var")):
            assert np.allclose(p[k].detach().numpy(), g[f"{prefix}after:{k}"], rtol=1e-14, atol=0), k
        if k.endswith(".num_batches_tracked"):
            assert int(p[k]) == int(g[f"{prefix}after:{k}"]), k


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_the_seeded_reference_cases(name):
    g = np.load(f"{GOLDEN}/image_resnet18_families_{name}.npz")
    cls, kwargs, training, shape, seed = CASES[name]
    m = getattr(I, cls)(**kwargs).train(training)
    state = O.hashed_state(m.state_dict(), seed)
    x = torch.from_numpy(O.hash_grid(seed, 50000, shape, 8, 2))
    assert float(x.sum()) == float(g["checksum:x"])
    for k, v in state.items():
        if k.endswith((".weight", ".bias", ".running_mean", ".running_var")):
            assert float(v.double().sum()) == float(g[f"checksum:{k}"]), k
    y, grads, p, names = run_oracle(m, state, x, seed, "Pyramid" in cls)
    check_step(g, y, grads, p, names, seed)
    if training:
        assert all(int(g[f"after:{k}"]) == 1 for k in state if k.endswith(".num_batches_tracked"))


@pytest.mark.parametrize("fam", sorted(LAYER0))
@pytest.mark.parametrize("mode", ["eval", "train"])
def test_oracle_reproduces_the_pretrained_layer0_fixtures(fam, mode):
    g = np.load(f"{GOLDEN}/image_resnet18_families_{fam}_layer0.npz")
    cls, shape, seed = LAYER0[fam]
    m = getattr(I, cls)().train(mode == "train")
    state = {k: torch.from_numpy(g[k]).double() if g[k].dtype != np.int64 else torch.from_numpy(g[k]).clone()
             for k in m.state_dict()}
    x = torch.from_numpy(O.hash_grid(seed, 50000, shape, 8, 2))
    assert float(x.sum()) == float(g["checksum:x"])
    y, grads, p, names = run_oracle(m, state, x, seed, False)
    check_step(g, y, grads, p, names, seed, f"{mode}:")


def _keys():
    return np.load(f"{GOLDEN}/image_resnet18_families_keys.npz")


def _checkpoint(which):
    """A zero state dict with the keys and shapes of a reference checkpoint."""
    k = _keys()
    shapes = [tuple(int(v) for v in s.strip("()").split(",") if v.strip()) for s in k[f"{which}:shapes"]]
    return {name: (torch.zeros(shape, dtype=torch.int64) if name.endswith("num_batches_tracked")
                   else torch.zeros(shape)) for name, shape in zip(k[f"{which}:keys"], shapes)}


@pytest.mark.parametrize("cls", CLASSES)
def test_state_dict_keys_are_the_reference_wrappers(cls):
    assert len(CLASSES) == 23
    m = getattr(I, cls)()
    assert list(m.state_dict()) == list(_keys()[f"keys:{cls}"])


def test_load_torchvision_resnet18_takes_the_legacy_checkpoint_and_torchvisions_keys():
    import torchvision
    sd = _checkpoint("imagenet")
    assert len(sd) == 102 and not any(k.endswith("num_batches_tracked") for k in sd)
    m = I.ResNet18Pyramid(weights=sd)
    assert all(float(p.detach().abs().sum()) == 0 for p in m.parameters())
    assert all(int(b.num_batches_tracked) == 0 for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d))
    # counters missing from a legacy checkpoint are left as they are
    m = I.ResNet18TruncatedLayer1()
    m.conv[0][1].num_batches_tracked.fill_(7)
    I.load_torchvision_resnet18(m, sd)
    assert int(m.conv[0][1].num_batches_tracked) == 7
    # torchvision's own state dict, counters included
    tv = torchvision.models.resnet18().state_dict()
    tv["layer3.1.bn2.num_batches_tracked"].fill_(5)
    m = I.ResNet18Layer3(weights=tv)
    assert int(m.conv[0][1].bn2.num_batches_tracked) == 5
    assert torch.equal(m.conv[0][0].conv1.weight, tv["layer3.0.conv1.weight"])
    assert torch.equal(I.ResNet18Layer0(weights=tv).conv[0][0].weight, tv["conv1.weight"])
    missing = dict(sd)
    missing.pop("fc.bias")
    with pytest.raises(KeyError, match="missing"):
        I.load_torchvision_resnet18(I.ResNet18Layer2(), missing)
    with pytest.raises(KeyError, match="unexpected"):
        I.load_torchvision_resnet18(I.ResNet18Layer2(), {**sd, "layer5.weight": torch.zeros(1)})


def test_load_cityscapes_resnet18_takes_exactly_the_sfsegnets_checkpoint():
    sd = _checkpoint("cityscapes")
    assert len(sd) == 138
    sd["layer2.0.downsample.1.num_batches_tracked"].fill_(3)
    full = I.CityscapesResNet18(weights=sd)
    assert int(full.layer2[0].downsample[1].num_batches_tracked) == 3
    m = I.CityscapesResNet18Layer2(weights=sd)
    assert int(m.conv[0][0].downsample[1].num_batches_tracked) == 3
    assert all(float(p.detach().abs().sum()) == 0 for p in m.parameters())
    I.load_cityscapes_resnet18(I.CityscapesResNet18Pyramid(), sd)
    with pytest.raises(KeyError, match="missing"):
        I.load_cityscapes_resnet18(I.CityscapesResNet18(), _checkpoint("other"))
    with pytest.raises(KeyError, match="unexpected"):
        I.CityscapesResNet18TruncatedLayer0(weights={**sd, "fc.weight": torch.zeros(1)})


def test_properties_frozen_and_train():
    m = I.ResNet18TruncatedLayer4(pretrained=True, foo=1)
    assert (m.input_nc, m.output_nc, m.conv_scale_factor, m.scale_factor) == (3, 512, 32, None)
    assert I.ResNet18TruncatedLayer0(scale_factor=-1).scale_factor == 4
    assert (I.ResNet18Layer1().input_nc, I.ResNet18Layer1().output_nc) == (64, 64)
    assert (I.CityscapesResNet18Layer0().output_nc, I.CityscapesResNet18Layer1().input_nc) == (128, 128)
    assert I.CityscapesResNet18Layer3().conv_scale_factor == 2
    p = I.CityscapesResNet18Pyramid(pretrained=False)
    assert p.scale_factor == 32 and p.extra_repr() == "scale_factor=32"
    with pytest.raises(AssertionError):
        I.ResNet18Pyramid(scale_factor=None)
    bn = m.conv[0][1]
    assert type(bn) is I.FusedBatchNorm2d and bn.momentum == 0.1 and m.conv[0][3].padding == 1
    assert I.CityscapesResNet18Layer0().conv[0][3].padding == 0
    for f in (I.ResNet18TruncatedLayer1(frozen=True), I.CityscapesResNet18(frozen=True)):
        assert f.frozen and not f.training and not any(p.requires_grad for p in f.parameters())
        f.train()
        assert not f.training and not any(mod.training for mod in f.modules())
        f.frozen = False
        f.train()
        assert f.training and all(p.requires_grad for p in f.parameters())
    c = I.CityscapesResNet18()
    assert [n for n, _ in c.named_children()] == ["layer0", "layer1", "layer2", "layer3", "layer4"]


def test_init_is_kaiming_fan_out():
    torch.manual_seed(0)
    m = I.CityscapesResNet18TruncatedLayer4()
    w = m.conv[4][0].conv2.weight
    assert abs(float(w.std()) / (2 / (9 * 512)) ** 0.5 - 1) < 0.01
    w = I.ResNet18TruncatedLayer0().conv[0][0].weight
    assert abs(float(w.std()) / (2 / (49 * 64)) ** 0.5 - 1) < 0.05
    assert all(float(b.weight.min()) == 1 and float(b.bias.abs().max()) == 0
               for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d))


def test_batchnorm_bookkeeping():
    """nn.BatchNorm2d's counter and momentum for the new families; mit_semseg's never moves."""
    bn = I.FusedBatchNorm2d(4)
    assert ops._bn_cfg(bn) == (True, 0.1, 1e-5) and int(bn.num_batches_tracked) == 1
    bn.momentum = None
    ops._bn_cfg(bn)
    assert ops._bn_cfg(bn) == (True, 1.0 / 3, 1e-5) and int(bn.num_batches_tracked) == 3
    bn.eval()
    ops._bn_cfg(bn)
    assert int(bn.num_batches_tracked) == 3
    sync = I.SynchronizedBatchNorm2d(4)
    assert ops._bn_cfg(sync) == (True, 0.001, 1e-5) and int(sync.num_batches_tracked) == 0


@pytest.mark.parametrize("cls,shape", [("CityscapesResNet18TruncatedLayer0", (1, 3, 4, 9)),
                                       ("CityscapesResNet18TruncatedLayer0", (1, 3, 9, 3)),
                                       ("CityscapesResNet18", (1, 3, 5, 5)), ("ResNet18TruncatedLayer4", (2, 3, 1, 1)),
                                       ("ResNet18TruncatedLayer4", (1, 3, 33, 33)),
                                       ("CityscapesResNet18Layer1", (1, 128, 1, 1))])
def test_size_checks_follow_torch(cls, shape):
    """ValueError exactly where the float64 restatement (torch's max_pool2d and F.batch_norm) raises, from the walk
    that runs before any launch."""
    m = getattr(I, cls)()
    B, _, H, W = shape

    def ours():
        for bn, h, w in m._bn_sizes(H, W):
            I._check_bn_values(bn, bn.training, B, h, w)

    fam, layers, prefixes = oracle_args(m)
    p = {k: v.double() if v.is_floating_point() else v.clone() for k, v in m.state_dict().items()}
    raised = []
    for fn in (ours, lambda: O.forward(torch.randn(*shape, dtype=torch.float64), p, fam, layers, True,
                                       prefixes=prefixes)):
        try:
            fn()
            raised.append(False)
        except (ValueError, RuntimeError):
            raised.append(True)
    assert raised[0] == raised[1]


def test_rn_pool_out():
    assert [ops.rn_pool_out(n, 1) for n in (1, 2, 7, 8)] == [ops.rn_out(n, 2) for n in (1, 2, 7, 8)]
    assert [ops.rn_pool_out(n, 0) for n in (3, 4, 5, 26)] == [1, 1, 2, 12]
    with pytest.raises(ValueError):
        ops.rn_pool_out(2, 0)
    with pytest.raises(ValueError):
        ops.rn_pool_out(8, 2)


def test_new_abi_entries_reject_bad_arguments_without_a_launch():
    lib = _lib.load_resnet()
    n0 = _lib.launch_count()
    buf = ctypes.c_void_p(16)   # never dereferenced: every call below fails its checks first
    rc = lib.dva_resnet_maxpool_pad(buf, 1, 8, 8, 4, 2, buf, buf, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_maxpool: padding must be 0 or 1"
    rc = lib.dva_resnet_maxpool_pad(buf, 1, 2, 8, 4, 0, buf, buf, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_maxpool: input smaller than one window"
    rc = lib.dva_resnet_maxpool_pad_bwd(buf, buf, 1, 8, 2, 4, 0, buf, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_maxpool_bwd: input smaller than one window"
    rc = lib.dva_resnet_maxpool_pad_bwd(buf, buf, 1, 8, 8, 4, -1, buf, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_maxpool_bwd: padding must be 0 or 1"
    rc = lib.dva_resnet_maxpool_pad(None, 1, 8, 8, 4, 0, None, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_maxpool: null pointer"
    rc = lib.dva_resnet_conv_bn_fwd(None, 1, 8, 8, 3, None, 64, 7, 1, 1, 1, 0.1, 1e-5, None, None, None, None, None,
                                    None, 0, None)
    assert rc == _lib.DVA_EINVAL and "unsupported shape (T 7, stride 1, dilation 1)" in _lib.last_error()
    rc = lib.dva_resnet_conv_dgrad(None, 1, 8, 8, 3, 64, None, 7, 2, 1, None, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_conv_dgrad: null pointer"
    rc = lib.dva_resnet_weight_prep(None, 64, 3, 5, None, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_weight_prep: T must be 1, 3 or 7"
    rc = lib.dva_resnet_weight_prep(None, 64, 3, 7, None, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_weight_prep: null pointer"
    assert _lib.launch_count() == n0
    # the 7x7 stem's weight gradient: Kd = 147 columns in 3 column tiles, one fp32 partial per split
    ws = lib.dva_resnet_wgrad_workspace_bytes(8, 512, 1024, 3, 64, 7, 2, 1)
    assert ws > 0 and ws % (64 * 147 * 4) == 0
    assert lib.dva_resnet_wgrad_workspace_bytes(1, 8, 8, 4, 8, 2, 1, 1) == 0
