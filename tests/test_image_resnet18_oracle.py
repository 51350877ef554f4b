"""The ADE20K ResNet-18 encoders without a GPU: the float64 restatement oracle/image_resnet18_oracle.py against the
fixtures made by executing the reference's wrappers (oracle/make_golden_image_resnet18.py), the classes' state-dict
keys against the reference's, load_mit_semseg_encoder against the checkpoint's layout, and the frozen / train()
semantics."""
import numpy as np
import pytest
import torch

from conftest import GOLDEN
from deepviewagg_b200.modules.multimodal.modalities import image as I
from oracle import image_resnet18_oracle as O

CLASSES = ["TruncatedLayer0", "TruncatedLayer1", "TruncatedLayer2", "TruncatedLayer3", "TruncatedLayer4", "Layer0",
           "Layer1", "Layer2", "Layer3", "Layer4", "Pyramid"]


def _keys():
    return np.load(f"{GOLDEN}/image_resnet18_keys.npz")


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_oracle_reproduces_the_pretrained_layer0_fixture(mode):
    g = np.load(f"{GOLDEN}/image_resnet18_layer0.npz")
    m = I.ADE20KResNet18TruncatedLayer0()
    p = {k: torch.from_numpy(g[k]).double() if g[k].dtype != np.int64 else torch.from_numpy(g[k])
         for k in m.state_dict()}
    names = [k for k, _ in m.named_parameters()]
    for k in names:
        p[k].requires_grad_(True)
    x = torch.from_numpy(g["x"]).requires_grad_(True)
    y = O.forward(x, p, m._LAYERS, mode == "train")
    grads = torch.autograd.grad(y, [x] + [p[k] for k in names], torch.from_numpy(g["gy"]))
    assert np.array_equal(y.detach().float().numpy(), g[f"{mode}:y"])
    assert abs(float(y.detach().norm()) / float(g[f"{mode}:y_norm"]) - 1) <= 1e-12
    assert abs(float(grads[0].norm()) / float(g[f"{mode}:gx_norm"]) - 1) <= 1e-12
    for k, gp in zip(names, grads[1:]):
        assert abs(float(gp.norm()) / float(g[f"{mode}:gnorm:{k}"]) - 1) <= 1e-12, k
    for k in m.state_dict():
        if "running_" in k:
            assert np.array_equal(p[k].numpy(), g[f"{mode}:after:{k}"]), k
    if mode == "eval":
        assert all(np.array_equal(g[f"eval:after:{k}"], g[k]) for k in m.state_dict() if "running_" in k)


@pytest.mark.parametrize("cls", CLASSES)
def test_state_dict_keys_are_the_reference_wrappers(cls):
    m = getattr(I, f"ADE20KResNet18{cls}")()
    assert list(m.state_dict()) == list(_keys()[f"keys:ADE20KResNet18{cls}"])


def test_load_mit_semseg_encoder_takes_exactly_the_checkpoint_layout():
    k = _keys()
    shapes = [tuple(int(v) for v in s.strip("()").split(",") if v.strip()) for s in k["ckpt_shapes"]]
    sd = {name: (torch.zeros(shape, dtype=torch.int64) if name.endswith("num_batches_tracked")
                 else torch.zeros(shape)) for name, shape in zip(k["ckpt_keys"], shapes)}
    assert len(sd) == 207
    m = I.ADE20KResNet18Pyramid(weights=sd)
    assert all(float(p.detach().abs().sum()) == 0 for p in m.parameters())
    I.load_mit_semseg_encoder(I.ADE20KResNet18Layer2(), sd)
    missing = dict(sd)
    missing.pop("layer4.1.bn2.weight")
    with pytest.raises(KeyError, match="missing"):
        I.load_mit_semseg_encoder(I.ADE20KResNet18Layer2(), missing)
    with pytest.raises(KeyError, match="unexpected"):
        I.load_mit_semseg_encoder(I.ADE20KResNet18Layer2(), {**sd, "fc.weight": torch.zeros(1)})


def test_properties_frozen_and_train():
    m = I.ADE20KResNet18TruncatedLayer4()
    assert (m.input_nc, m.output_nc, m.conv_scale_factor, m.scale_factor) == (3, 512, 8, None)
    assert m.training and all(p.requires_grad for p in m.parameters()) and m.extra_repr() == ""
    bn = m.conv[0][1]
    assert bn.momentum == 0.001 and bn._running_iter.shape == (1,)
    assert I.ADE20KResNet18TruncatedLayer2(scale_factor=-1).scale_factor == 8
    assert I.ADE20KResNet18Layer1().input_nc == 128 and I.ADE20KResNet18Layer1().conv_scale_factor == 1
    p = I.ADE20KResNet18Pyramid(foo=1)
    assert p.scale_factor == 8 and p.extra_repr() == "scale_factor=8"
    with pytest.raises(AssertionError):
        I.ADE20KResNet18Pyramid(scale_factor=None)
    f = I.ADE20KResNet18TruncatedLayer1(frozen=True)
    assert f.frozen and not f.training and not any(p.requires_grad for p in f.parameters())
    f.train()
    assert not f.training and not any(mod.training for mod in f.modules())
    f.frozen = False
    f.train()
    assert f.training and all(p.requires_grad for p in f.parameters())


def test_init_is_mit_semsegs():
    torch.manual_seed(0)
    m = I.ADE20KResNet18TruncatedLayer4()
    w = m.conv[4][0].conv2.weight
    assert abs(float(w.std()) / (2 / (9 * 512)) ** 0.5 - 1) < 0.01
    assert all(float(b.weight.min()) == 1 and float(b.bias.abs().max()) == 0
               for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d))


def test_fused_modules_do_not_run_alone():
    m = I.ADE20KResNet18TruncatedLayer0()
    for mod in (m.conv[0][0], m.conv[0][1], m.conv[0][2], m.conv[0][9]):
        with pytest.raises(NotImplementedError):
            mod(torch.zeros(1, mod.in_channels if hasattr(mod, "in_channels") else 64, 4, 4))


@pytest.mark.parametrize("cls,shape", [("TruncatedLayer4", (1, 3, 16, 16)), ("Layer2", (1, 64, 3, 3)),
                                       ("TruncatedLayer4", (1, 3, 8, 8)), ("Layer1", (1, 128, 1, 1))])
def test_one_value_per_channel_check_follows_torch(cls, shape):
    """The sizes each BatchNorm sees (the downsample runs beside conv1, not after it): train mode raises ValueError
    exactly where the float64 restatement (torch's F.batch_norm) raises."""
    m = getattr(I, f"ADE20KResNet18{cls}")()
    B, _, H, W = shape
    sizes = {id(bn): (h, w) for bn, h, w in m._bn_sizes(H, W)}
    assert len(sizes) == sum(isinstance(b, torch.nn.BatchNorm2d) for b in m.modules())
    p = {k: v.double() if v.is_floating_point() else v for k, v in m.state_dict().items()}
    try:
        O.forward(torch.randn(*shape, dtype=torch.float64), p, m._LAYERS, True)
        torch_raises = False
    except ValueError:
        torch_raises = True
    assert torch_raises == any(B * h * w <= 1 for h, w in sizes.values())


CASES = {  # oracle/make_golden_image_resnet18.py:CASES
    "tl4_train": ("TruncatedLayer4", {}, True, (2, 3, 61, 45), 1),
    "layer3_train": ("Layer3", {}, True, (2, 128, 13, 11), 2),
    "layer2_eval": ("Layer2", {}, False, (1, 64, 15, 18), 3),
    "tl2_sf8_eval": ("TruncatedLayer2", {"scale_factor": -1}, False, (2, 3, 21, 30), 4),
    "pyramid_sf2_train": ("Pyramid", {"scale_factor": 2}, True, (2, 3, 24, 40), 5),
}


def case_inputs(name):
    """(module, float64 state, x, gy) of a seeded case, regenerated from the integer-hash generator."""
    cls, kwargs, training, shape, seed = CASES[name]
    m = getattr(I, f"ADE20KResNet18{cls}")(**kwargs).train(training)
    state = O.hashed_state(m.state_dict(), seed)
    x = torch.from_numpy(O.hash_grid(seed, 50000, shape, 8, 2))
    return m, state, x, seed


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_the_seeded_reference_cases(name):
    g = np.load(f"{GOLDEN}/image_resnet18_{name}.npz")
    m, state, x, seed = case_inputs(name)
    assert float(x.sum()) == float(g["checksum:x"])
    for k, v in state.items():
        if k.endswith((".weight", ".bias", ".running_mean", ".running_var")):
            assert float(v.double().sum()) == float(g[f"checksum:{k}"]), k
            assert torch.equal(v.float().double(), v), k            # the grid is exact in float32
    p = {k: v.clone() for k, v in state.items()}
    names = [k for k, _ in m.named_parameters()]
    for k in names:
        p[k].requires_grad_(True)
    x.requires_grad_(True)
    y = O.forward(x, p, m._LAYERS, m.training, m.scale_factor, isinstance(m, I.ADE20KResNet18Pyramid))
    gy = torch.from_numpy(O.hash_grid(seed, 60000, tuple(y.shape), 8, 3))
    grads = torch.autograd.grad(y, [x] + [p[k] for k in names], gy)
    u = 2.0 ** -24
    assert np.abs(y.detach().float().numpy() - g["y"]).max() <= u * np.abs(g["y"]).max()
    assert np.abs(grads[0].float().numpy() - g["gx"]).max() <= u * np.abs(g["gx"]).max()
    assert abs(float(y.detach().norm()) / float(g["y_norm"]) - 1) <= 1e-12
    assert abs(float(grads[0].norm()) / float(g["gx_norm"]) - 1) <= 1e-12
    for tag, (k, gp) in enumerate(zip(names, grads[1:])):
        assert abs(float(gp.norm()) / float(g[f"gnorm:{k}"]) - 1) <= 1e-12, k
        proj = float((gp * O.projection(seed, tag, tuple(gp.shape))).sum())
        assert abs(proj - float(g[f"gproj:{k}"])) <= 1e-12 * float(g[f"gnorm:{k}"]) * gp.numel() ** 0.5, k
    for k in state:
        if k.endswith((".running_mean", ".running_var")):
            assert np.allclose(p[k].detach().numpy(), g[f"after:{k}"], rtol=1e-14, atol=0), k
