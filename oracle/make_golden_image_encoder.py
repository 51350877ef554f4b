"""Fixtures of the from-scratch image encoder, made by EXECUTING the reference's ResNetDown
(torch_points3d/modules/multimodal/modalities/image.py), loaded by file path in float64 on the CPU.

    PYTORCH_JIT=0 python -m oracle.make_golden_image_encoder      # writes tests/golden/image_encoder_*.npz

What the file needs that is not there:
  * mit_semseg.* (the pretrained encoders' package, imported at module level) and torch_points3d.utils.config
    (is_list, fetch_arguments_from_list) are stubbed; torch_points3d.core.common_modules gets Seq and Identity;
  * the reference's Conv2dWS.forward calls self._conv_forward(x, weights), torch 1.7's signature.  Since torch 1.8
    _conv_forward takes the bias as a third argument and the call raises TypeError, so nn.Conv2d._conv_forward is
    wrapped to restore the 1.7 behaviour: with two arguments it uses self.bias.

Layout: the five chained stages of the shipped no3d / sparseconv3d GroupNorm encoders (N = [0, 2, 2, 2, 2], kernels
[3, 2, 2, 2, 2], strides [1, 2, 2, 2, 2], paddings [1, 0, 0, 0, 0], 4 input channels) at in_feat = 4, so the
GroupNorms have 1 group (4, 8, 16 channels) and 2 groups (32 channels).  Cases: B = 2 at 41 x 35 (every stage >= 2
wide: 41x35, 20x17, 10x8, 5x4, 2x2) and B = 1 at 48 x 64.  Each file holds the input, the parameters (GroupNorm
affine parameters perturbed from 1 / 0), an upstream gradient, the output, the gradient of the input and of every
parameter, and the state-dict keys of every stage."""
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

from oracle import ref_loader

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
IN_FEAT = 4
CHANNELS = [[4, IN_FEAT], [IN_FEAT, IN_FEAT], [IN_FEAT, 2 * IN_FEAT], [2 * IN_FEAT, 4 * IN_FEAT],
            [4 * IN_FEAT, 8 * IN_FEAT]]
N = [0, 2, 2, 2, 2]
KERNEL = [3, 2, 2, 2, 2]
STRIDE = [1, 2, 2, 2, 2]
PADDING = [1, 0, 0, 0, 0]
CASES = {"b2": (2, 41, 35, 0), "b1": (1, 48, 64, 1)}


class _Seq(nn.Sequential):
    def __init__(self):
        super().__init__()
        self._num_modules = 0

    def append(self, module):
        self.add_module(str(self._num_modules), module)
        self._num_modules += 1
        return self


class _Identity(nn.Module):
    def forward(self, x):
        return x


def _is_list(x):
    return isinstance(x, list)


def _fetch_arguments_from_list(*args, **kwargs):
    raise NotImplementedError("not used by ResNetDown")


_ORIG_CONV_FORWARD = nn.Conv2d._conv_forward
_MISSING = object()


def _conv_forward_torch17(self, input, weight, bias=_MISSING):
    return _ORIG_CONV_FORWARD(self, input, weight, self.bias if bias is _MISSING else bias)


def load_reference_image():
    """The reference's modalities/image.py, executed with the stubs and the torch 1.7 _conv_forward shim."""
    name = "torch_points3d.modules.multimodal.modalities.image"
    if name in sys.modules:
        return sys.modules[name]
    for pkg in ["torch_points3d", "torch_points3d.utils", "torch_points3d.core", "torch_points3d.modules",
                "torch_points3d.modules.multimodal", "torch_points3d.modules.multimodal.modalities", "mit_semseg",
                "mit_semseg.lib"]:
        ref_loader._stub(pkg)
    cfg = ref_loader._stub("torch_points3d.utils.config")
    cfg.is_list, cfg.fetch_arguments_from_list = _is_list, _fetch_arguments_from_list
    cfg.__all__ = ["is_list", "fetch_arguments_from_list"]
    cm = ref_loader._stub("torch_points3d.core.common_modules")
    cm.Seq, cm.Identity = _Seq, _Identity
    ref_loader._stub("mit_semseg.config").cfg = types.SimpleNamespace()
    ref_loader._stub("mit_semseg.models").ModelBuilder = type("ModelBuilder", (), {})
    ref_loader._stub("mit_semseg.lib.nn").SynchronizedBatchNorm2d = nn.BatchNorm2d
    nn.Conv2d._conv_forward = _conv_forward_torch17
    return ref_loader._load(name, "torch_points3d/modules/multimodal/modalities/image.py")


def stage_kwargs(i, channels=CHANNELS):
    return dict(down_conv_nn=channels[i], kernel_size=KERNEL[i], stride=STRIDE[i], padding=PADDING[i], N=N[i],
                block="ResBlock", normalization="GroupNorm", weight_standardization=True)


def build_reference(seed):
    image = load_reference_image()
    torch.manual_seed(seed)
    stages = [image.ResNetDown(**stage_kwargs(i)).double() for i in range(len(CHANNELS))]
    gen = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for st in stages:
            for m in st.modules():
                if isinstance(m, nn.GroupNorm):
                    m.weight.copy_(1 + 0.2 * torch.randn(m.weight.shape, generator=gen, dtype=torch.float64))
                    m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=gen, dtype=torch.float64))
    return stages


def make_case(B, H, W, seed):
    stages = build_reference(seed)
    gen = torch.Generator().manual_seed(seed + 200)
    x = torch.randn(B, 4, H, W, generator=gen, dtype=torch.float64).requires_grad_(True)
    y = x
    for st in stages:
        y = st(y)
    gy = torch.randn(y.shape, generator=gen, dtype=torch.float64)
    params = [p for st in stages for p in st.parameters()]
    grads = torch.autograd.grad(y, [x] + params, gy)
    out = {"x": x.detach().numpy(), "gy": gy.numpy(), "y": y.detach().numpy(), "gx": grads[0].numpy()}
    gi = iter(grads[1:])
    for i, st in enumerate(stages):
        out[f"keys{i}"] = np.array(list(st.state_dict().keys()))
        for k, p in st.named_parameters():
            out[f"p{i}:{k}"] = p.detach().numpy()
            out[f"g{i}:{k}"] = next(gi).numpy()
    return out


def main():
    os.environ.setdefault("PYTORCH_JIT", "0")
    for name, (B, H, W, seed) in CASES.items():
        d = make_case(B, H, W, seed)
        path = os.path.join(OUT, f"image_encoder_{name}.npz")
        np.savez_compressed(path, **d)
        print(path, d["y"].shape, os.path.getsize(path))


if __name__ == "__main__":
    main()
