"""The from-scratch image encoder without a GPU: the float64 oracle (oracle/image_encoder_oracle.py) reproduces the
fixtures made by executing the reference's ResNetDown (oracle/make_golden_image_encoder.py), and the executed
reference itself where it is available; our ResNetDown has the reference's state-dict keys and shapes for every
stage of every shipped GroupNorm config, and rejects what it does not support."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from deepviewagg_b200.modules.multimodal.modalities.image import ResNetDown
from oracle import image_encoder_oracle as O
from oracle import make_golden_image_encoder as MG
from oracle import ref_loader

CASES = sorted(MG.CASES)


def load_case(name):
    z = np.load(os.path.join(GOLDEN, f"image_encoder_{name}.npz"), allow_pickle=False)
    return {k: z[k] for k in z.files}


def stage_dicts(d, requires_grad=False):
    sds = []
    for i in range(len(MG.CHANNELS)):
        sd = {k.split(":", 1)[1]: torch.from_numpy(v).requires_grad_(requires_grad)
              for k, v in d.items() if k.startswith(f"p{i}:")}
        sds.append(sd)
    return sds


def oracle_run(d):
    sds = stage_dicts(d, requires_grad=True)
    x = torch.from_numpy(d["x"]).requires_grad_(True)
    y = O.encoder(x, [(sd, MG.KERNEL[i], MG.STRIDE[i], MG.PADDING[i]) for i, sd in enumerate(sds)])
    params = [(i, k, p) for i, sd in enumerate(sds) for k, p in sd.items()]
    grads = torch.autograd.grad(y, [x] + [p for _, _, p in params], torch.from_numpy(d["gy"]))
    return y.detach(), grads[0], {f"g{i}:{k}": g for (i, k, _), g in zip(params, grads[1:])}


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_fixtures(name):
    d = load_case(name)
    y, gx, gp = oracle_run(d)
    np.testing.assert_allclose(y.numpy(), d["y"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(gx.numpy(), d["gx"], rtol=1e-9, atol=1e-12)
    assert set(gp) == {k for k in d if k.startswith("g") and ":" in k}
    for k, g in gp.items():
        np.testing.assert_allclose(g.numpy(), d[k], rtol=1e-9, atol=1e-10, err_msg=k)


@pytest.mark.needs_reference
@pytest.mark.skipif(not ref_loader.available(), reason="reference not available")
def test_oracle_equals_executed_reference():
    os.environ.setdefault("PYTORCH_JIT", "0")
    d = MG.make_case(1, 33, 40, 7)
    y, gx, gp = oracle_run(d)
    np.testing.assert_allclose(y.numpy(), d["y"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(gx.numpy(), d["gx"], rtol=1e-9, atol=1e-12)
    for k, g in gp.items():
        np.testing.assert_allclose(g.numpy(), d[k], rtol=1e-9, atol=1e-10, err_msg=k)


@pytest.mark.parametrize("name", CASES)
def test_fixture_state_dict_keys_match_ours(name):
    d = load_case(name)
    for i in range(len(MG.CHANNELS)):
        ours = ResNetDown(**MG.stage_kwargs(i))
        assert list(ours.state_dict().keys()) == list(d[f"keys{i}"])
        ours.load_state_dict({k: torch.from_numpy(d[f"p{i}:{k}"]).float() for k in d[f"keys{i}"]}, strict=True)


# ---- every ResNetDown of the shipped GroupNorm configs (conf/models/segmentation/multimodal/*.yaml)
def _resolve(v, consts):
    if isinstance(v, list):
        return [_resolve(u, consts) for u in v]
    if isinstance(v, str) and v not in ("ResBlock", "GroupNorm", "reflect"):
        expr = re.sub(r"[A-Za-z_]\w*", lambda m: str(consts.get(m.group(0), m.group(0))), v)
        return int(eval(expr, {"__builtins__": {}}))
    return v


def shipped_groupnorm_encoders():
    import yaml
    root = os.path.join(ref_loader.REFERENCE_ROOT, "conf", "models", "segmentation", "multimodal")
    found = []
    for f in ("no3d.yaml", "sparseconv3d.yaml"):
        for model, cfg in yaml.safe_load(open(os.path.join(root, f))).items():
            if not isinstance(cfg, dict):
                continue
            # a model without its own constants takes the widths most configs define
            consts = {"in_feat_img": 4, "in_feat": 32, "strided_k": 2, "strided_s": 2, "strided_p": 0, **(cfg.get("define_constants", {}) or {})}

            def walk(o):
                if isinstance(o, dict):
                    if o.get("module_name") == "ResNetDown" and o.get("normalization") == "GroupNorm":
                        found.append((f, model, o, consts))
                    for v in o.values():
                        walk(v)
                elif isinstance(o, list):
                    for v in o:
                        walk(v)
            walk(cfg)
    return found


def stage_args(opt, consts):
    """The per-stage kwargs of the compact format (fetch_arguments_from_list: plural list names are indexed)."""
    nn_ = _resolve(opt["down_conv_nn"], consts)
    stages = []
    for i in range(len(nn_)):
        kw = {"down_conv_nn": nn_[i]}
        for k, v in opt.items():
            if k in ("module_name", "down_conv_nn"):
                continue
            v = _resolve(v, consts)
            kw[k] = v[i] if isinstance(v, list) else v
        stages.append(kw)
    return stages


@pytest.mark.needs_reference
@pytest.mark.skipif(not ref_loader.available(), reason="reference not available")
def test_every_shipped_groupnorm_stage_has_the_reference_state_dict():
    os.environ.setdefault("PYTORCH_JIT", "0")
    image = MG.load_reference_image()
    encoders = shipped_groupnorm_encoders()
    assert len(encoders) == 43
    n = 0
    for f, model, opt, consts in encoders:
        for kw in stage_args(opt, consts):
            ref = image.ResNetDown(**kw)
            ours = ResNetDown(**kw)
            rs, os_ = ref.state_dict(), ours.state_dict()
            assert list(rs) == list(os_), (f, model, kw)
            assert all(rs[k].shape == os_[k].shape for k in rs), (f, model, kw)
            ours.load_state_dict(rs, strict=True)
            n += 1
    assert n > 43


BASE = dict(down_conv_nn=[8, 16], kernel_size=2, stride=2, padding=0, N=1, block="ResBlock",
            normalization="GroupNorm", weight_standardization=True)


@pytest.mark.parametrize("kw, word", [
    ({"normalization": "BatchNorm2d"}, "normalization"),
    ({"weight_standardization": False}, "weight_standardization"),
    ({"block": "BottleneckBlock"}, "block"),
    ({"padding_mode": "zeros"}, "padding_mode"),
    ({"dilation": 2}, "dilation"),
    ({"kernel_size": 3, "stride": 2, "padding": 1}, "kernel_size"),
    ({"kernel_size": 1, "stride": 1, "padding": 0}, "kernel_size"),
])
def test_unsupported_kwargs_raise(kw, word):
    with pytest.raises(NotImplementedError, match=word):
        ResNetDown(**{**BASE, **kw})


def test_extra_kwargs_swallowed_and_pass_through():
    ResNetDown(**BASE, index=3)
    ident = ResNetDown(down_conv_nn=[-1, -1])
    x = torch.zeros(1, 3, 4, 4)
    assert ident(x, True) is x


def test_cpu_tensors_and_small_images_raise():
    m = ResNetDown(**BASE)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        m(torch.zeros(1, 8, 8, 8))
    with pytest.raises(ValueError, match=">= 2"):
        m.output_hw(3, 8)     # 2x2 conv_in -> 1 x 4, then the blocks' reflect pad
    assert m.output_hw(5, 9) == (2, 4)


def test_standardize_weights_takes_the_fan_in_root_in_float32():
    from deepviewagg_b200.modules.multimodal.modalities.image import standardize_weights
    w = torch.randn(8, 32, 3, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    ours = standardize_weights(w)
    torch.testing.assert_close(ours, O.standardize(w), rtol=1e-13, atol=1e-15)
    # with the root taken in float64 the result would be ~5e-8 relative away
    fp64_root = standardize_weights(w, scaled=False) / 32 ** 0.5
    assert float(((ours - fp64_root) / fp64_root).abs().max()) > 1e-9


@pytest.mark.needs_reference
@pytest.mark.skipif(not ref_loader.available(), reason="reference not available")
def test_standardize_weights_equals_executed_reference():
    from deepviewagg_b200.modules.multimodal.modalities.image import standardize_weights
    os.environ.setdefault("PYTORCH_JIT", "0")
    image = MG.load_reference_image()
    for dt in (torch.float32, torch.float64):
        w = torch.randn(16, 32, 2, 2, generator=torch.Generator().manual_seed(4)).to(dt)
        assert torch.equal(standardize_weights(w), image.standardize_weights(w))
