"""Fixtures of the image UNet, made by EXECUTING the reference's UNet (torch_points3d/modules/multimodal/modalities/
image.py: module tree, _build_module, forward) in float64 on the CPU.

    PYTORCH_JIT=0 python -m oracle.make_golden_image_unet      # writes tests/golden/image_unet_*.npz

It reuses the stubs and the torch 1.7 _conv_forward shim of make_golden_image_encoder.py, and adds:
  * the reference's own fetch_arguments_from_list (torch_points3d/utils/config.py), loaded with hydra stubbed and
    omegaconf's DictConfig / ListConfig replaced by dict / list subclasses (DictConfig with attribute access);
  * a shim for ConvTranspose2dWS.forward: it calls self._output_padding(x, output_size, stride, padding,
    kernel_size), torch < 1.12's signature; torch now also requires num_spatial_dims, and the call raises TypeError.
    The shim passes num_spatial_dims = 2.

Topologies, at in_feat = 4, in_feat_img = 4 and 13 classes: "unet5" is the 5 down / 5 up shape of
Res16UNet21-15_light (the last up-stage [f, 0, f] is a stride-1 3x3 without skip), "unet4" the 5 down / 4 up shape
of RGB_D32_mean_view; both end in last_conv (1x1 to 13 classes).  Cases: unet5 with B = 2 at 48 x 32, unet4 with
B = 1 at 64 x 80.
Each file holds the input, the parameters (GroupNorm affine parameters perturbed from 1 / 0), an upstream gradient,
the output, the gradients of the input and of every parameter, and the state-dict keys.  To keep the files small,
the input, the upstream gradient and the parameters lie on coarse binary grids (multiples of 2^-4, 2^-2 and 2^-8),
so float32 holds them exactly and they compress; the reference runs on them in float64, and its output and gradients
are stored rounded to float32, each with its float64 2-norm so that the oracle stays pinned beyond float32.  The
parameters and their gradients are packed in state-dict order into one flat array each ("params", "grads"), with
"shapes" (JSON) and "grad_norms" per key.

image_unet_configs.npz: for every UNet config of conf/models/segmentation/multimodal/no3d.yaml (define_constants and
N_CLS = 13 substituted), its resolved image options as JSON, its normalization, and the reference's state-dict keys
and shapes at full width; also what the reference does with the two options it cannot run (persistent dropout in
last_conv, ConvTranspose2dWS without the shim), and standardize_weights on a transposed weight."""
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import yaml

from oracle import ref_loader
from oracle import make_golden_image_encoder as MG

OUT = MG.OUT
F = 4
N_CLS = 13
DOWN = dict(module_name="ResNetDown", block="ResBlock", normalization="GroupNorm", weight_standardization=True,
            N=[0, 2, 2, 2, 2], stride=[1, 2, 2, 2, 2], kernel_size=[3, 2, 2, 2, 2], padding=[1, 0, 0, 0, 0],
            down_conv_nn=[[4, F], [F, F], [F, 2 * F], [2 * F, 4 * F], [4 * F, 8 * F]])
UP5 = dict(module_name="ResNetUp", block="ResBlock", normalization="GroupNorm", weight_standardization=True, N=1,
           kernel_size=[2, 2, 2, 2, 3], stride=[2, 2, 2, 2, 1], padding=[0, 0, 0, 0, 1],
           up_conv_nn=[[8 * F, 4 * F, 4 * F], [4 * F, 2 * F, 3 * F], [3 * F, F, 2 * F], [2 * F, F, F], [F, 0, F]])
UP4 = dict(module_name="ResNetUp", block="ResBlock", normalization="GroupNorm", weight_standardization=True, N=1,
           kernel_size=[2, 2, 2, 2], stride=[2, 2, 2, 2], padding=[0, 0, 0, 0],
           up_conv_nn=[[8 * F, 4 * F, 4 * F], [4 * F, 2 * F, 3 * F], [3 * F, F, 2 * F], [2 * F, F, F]])
LAST = dict(input_nc=F, output_nc=N_CLS)
TOPOLOGIES = {"unet5": dict(down_conv=DOWN, up_conv=UP5, last_conv=LAST),
              "unet4": dict(down_conv=DOWN, up_conv=UP4, last_conv=LAST)}
# (topology, B, H, W, seed)
CASES = {"unet5_b2": ("unet5", 2, 48, 32, 0), "unet4_b1": ("unet4", 1, 64, 80, 1)}


class DictConfig(dict):
    """omegaconf.DictConfig stand-in: a dict with attribute access."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


class ListConfig(list):
    pass


def to_cfg(o):
    if isinstance(o, dict):
        return DictConfig({k: to_cfg(v) for k, v in o.items()})
    if isinstance(o, list):
        return ListConfig([to_cfg(v) for v in o])
    return o


_ORIG_OUTPUT_PADDING = nn.ConvTranspose2d._output_padding


def _output_padding_torch111(self, input, output_size, stride, padding, kernel_size, num_spatial_dims=2,
                             dilation=None):
    return _ORIG_OUTPUT_PADDING(self, input, output_size, stride, padding, kernel_size, num_spatial_dims, dilation)


def load_reference_config():
    """The reference's torch_points3d/utils/config.py with hydra and omegaconf stubbed."""
    ref_loader._stub("hydra").initialize = ref_loader._stub("hydra").compose = None
    oc = ref_loader._stub("omegaconf")
    oc.OmegaConf = type("OmegaConf", (), {})
    ref_loader._stub("omegaconf.listconfig").ListConfig = ListConfig
    ref_loader._stub("omegaconf.dictconfig").DictConfig = DictConfig
    for pkg in ["torch_points3d", "torch_points3d.utils"]:
        ref_loader._stub(pkg)
    ref_loader._stub("torch_points3d.utils.enums").ConvolutionFormat = type("ConvolutionFormat", (), {})
    ref_loader._stub("torch_points3d.utils.debugging_vars").DEBUGGING_VARS = {}
    return ref_loader._load("torch_points3d.utils.config_reference", "torch_points3d/utils/config.py")


def load_reference():
    """(image module, config module): the reference's image.py executing the reference's own
    fetch_arguments_from_list and is_list."""
    cfg = load_reference_config()
    image = MG.load_reference_image()
    image.fetch_arguments_from_list, image.is_list = cfg.fetch_arguments_from_list, cfg.is_list
    return image, cfg


def perturb(net, seed):
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, nn.GroupNorm):
                m.weight.copy_(1 + 0.2 * torch.randn(m.weight.shape, generator=gen, dtype=torch.float64))
                m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=gen, dtype=torch.float64))


def on_grid(t, bits):
    """t rounded to a multiple of 2^-bits: exact in float32."""
    return torch.round(t * 2.0 ** bits) / 2.0 ** bits


def make_case(image, topo, B, H, W, seed):
    torch.manual_seed(seed)
    net = image.UNet(to_cfg(TOPOLOGIES[topo])).double()
    perturb(net, seed + 100)
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(on_grid(p, 8))
    gen = torch.Generator().manual_seed(seed + 200)
    x = on_grid(torch.randn(B, 4, H, W, generator=gen, dtype=torch.float64), 4).requires_grad_(True)
    nn.ConvTranspose2d._output_padding = _output_padding_torch111
    try:
        y = net(x)
    finally:
        nn.ConvTranspose2d._output_padding = _ORIG_OUTPUT_PADDING
    gy = on_grid(torch.randn(y.shape, generator=gen, dtype=torch.float64), 2)
    names = [k for k, _ in net.named_parameters()]
    grads = torch.autograd.grad(y, [x] + [p for _, p in net.named_parameters()], gy)
    params = [p for _, p in net.named_parameters()]
    assert names == list(net.state_dict().keys())
    out = {"x": x.detach().float().numpy(), "gy": gy.float().numpy(), "keys": np.array(names),
           "shapes": np.array([json.dumps(list(p.shape)) for p in params]),
           "params": torch.cat([p.detach().reshape(-1) for p in params]).float().numpy(),
           "grads": torch.cat([g.reshape(-1) for g in grads[1:]]).float().numpy(),
           "grad_norms": np.array([float(g.norm()) for g in grads[1:]], dtype=np.float64)}
    for name, t in (("y", y), ("gx", grads[0])):
        out[name] = t.detach().float().numpy()
        out[f"norm_{name}"] = np.float64(t.detach().norm())
    return out


def resolve(o, constants):
    """define_constants (and N_CLS) substituted into the config's arithmetic strings."""
    if isinstance(o, dict):
        return {k: resolve(v, constants) for k, v in o.items()}
    if isinstance(o, list):
        return [resolve(v, constants) for v in o]
    if isinstance(o, str):
        try:
            return eval(o, {}, dict(constants))
        except (NameError, SyntaxError):
            return o
    return o


def shipped_configs():
    path = os.path.join(ref_loader.REFERENCE_ROOT, "conf/models/segmentation/multimodal/no3d.yaml")
    models = yaml.safe_load(open(path))
    for name, m in models.items():
        if not isinstance(m, dict) or "down_conv" not in m or "image" not in (m["down_conv"] or {}):
            continue
        img = m["down_conv"]["image"]
        if img.get("up_conv") is None:
            continue
        constants = dict(m.get("define_constants") or {}, N_CLS=N_CLS)
        opt = resolve({k: img[k] for k in ("down_conv", "up_conv", "innermost", "last_conv") if k in img}, constants)
        yield name, opt


def make_configs(image):
    out, names = {}, []
    for i, (name, opt) in enumerate(shipped_configs()):
        net = image.UNet(to_cfg(opt))
        sd = net.state_dict()
        names.append(name)
        out[f"opt{i}"] = np.array(json.dumps(opt))
        out[f"norm{i}"] = np.array(opt["down_conv"].get("normalization", ""))
        out[f"keys{i}"] = np.array(list(sd.keys()))
        out[f"shapes{i}"] = np.array([json.dumps(list(v.shape)) for v in sd.values()])
    out["names"] = np.array(names)
    # what the reference does with persistent dropout in last_conv: UNet.forward calls self.last(x) without reset
    torch.manual_seed(0)
    net = image.UNet(to_cfg(dict(TOPOLOGIES["unet4"], last_conv=dict(LAST, in_drop=0.5, persistent_drop=True))))
    net = net.double().train()
    x = torch.randn(1, 4, 32, 32, dtype=torch.float64)
    nn.ConvTranspose2d._output_padding = _output_padding_torch111
    try:
        net(x)
        out["persistent_drop_error"] = np.array("")
    except TypeError as e:
        out["persistent_drop_error"] = np.array(f"TypeError: {e}")
    finally:
        nn.ConvTranspose2d._output_padding = _ORIG_OUTPUT_PADDING
    # ConvTranspose2dWS.forward without the shim
    ct = image.ConvTranspose2dWS(4, 8, kernel_size=2, stride=2).double()
    try:
        ct(torch.randn(1, 4, 4, 4, dtype=torch.float64))
        out["convt_error"] = np.array("")
    except TypeError as e:
        out["convt_error"] = np.array(f"TypeError: {e}")
    # standardize_weights on transposed weights [C_in, C_out, R, S], fp32 and fp64
    gen = torch.Generator().manual_seed(7)
    for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        for shape in ((48, 16, 3, 3), (32, 32, 2, 2)):
            w = torch.randn(shape, generator=gen, dtype=dt)
            key = f"ws_{tag}_{'x'.join(map(str, shape))}"
            out[key + "_w"] = w.numpy()
            out[key + "_ref"] = image.standardize_weights(w).numpy()
    return out


def main():
    os.environ.setdefault("PYTORCH_JIT", "0")
    image, _ = load_reference()
    for name, (topo, B, H, W, seed) in CASES.items():
        d = make_case(image, topo, B, H, W, seed)
        path = os.path.join(OUT, f"image_unet_{name}.npz")
        np.savez_compressed(path, **d)
        print(path, d["y"].shape, os.path.getsize(path))
    d = make_configs(image)
    path = os.path.join(OUT, "image_unet_configs.npz")
    np.savez_compressed(path, **d)
    print(path, list(d["names"]), str(d["persistent_drop_error"]), str(d["convt_error"]), os.path.getsize(path))


if __name__ == "__main__":
    main()
