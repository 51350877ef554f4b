"""Fixtures of the ADE20K ResNet-18 encoders, made by EXECUTING the reference's ADE20KResNet18* wrappers
(torch_points3d/modules/multimodal/modalities/image.py:793-956), loaded by file path in float64 on the CPU.

    PYTORCH_JIT=0 python -m oracle.make_golden_image_resnet18      # writes tests/golden/image_resnet18_*.npz

What the file needs that is not there: mit_semseg is stubbed by a restatement of what the wrappers use --
resnet18 with the deep stem, BasicBlock, ResnetDilated / _nostride_dilate (dilate_scale 8) and the single-device
SynchronizedBatchNorm2d (momentum 0.001, the three extra buffers, an F.batch_norm forward) -- and MITCfg.merge_from_file
is stubbed to the values of resnet18dilated-ppm_deepsup.yaml the wrappers read.  The stubbed
ModelBuilder.build_encoder loads the reference's encoder_epoch_20.pth with strict=True, which proves that the
restated tree is the checkpoint's.

Files:
  image_resnet18_keys.npz    the checkpoint's key names and shapes (no values), and the state-dict keys of the
                             reference wrapper of every class;
  image_resnet18_layer0.npz  the checkpoint's real layer0 parameters and running stats under the wrapper's keys
                             (conv.0.*), and an eval-mode and a train-mode step of TruncatedLayer0 on them.
  image_resnet18_<case>.npz  seeded cases (CASES): parameters, running stats, input and upstream gradient from the
                             integer-hash generator of oracle/image_resnet18_oracle.py (a coarse binary grid, not
                             torch's RNG; per-tensor checksums stored), one step of the reference wrapper in float64:
                             the output and the input gradient rounded to float32 with their float64 norms, the
                             running stats after the step, and per parameter the gradient norm and its projection on
                             a fixed +-1 direction.
tests/test_image_resnet18_oracle.py checks oracle/image_resnet18_oracle.py against every fixture."""
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import image_resnet18_oracle as O
from oracle import ref_loader
from oracle.make_golden_image_encoder import _Identity, _Seq, _fetch_arguments_from_list, _is_list

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
CLASSES = ["ADE20KResNet18TruncatedLayer0", "ADE20KResNet18TruncatedLayer1", "ADE20KResNet18TruncatedLayer2",
           "ADE20KResNet18TruncatedLayer3", "ADE20KResNet18TruncatedLayer4", "ADE20KResNet18Layer0",
           "ADE20KResNet18Layer1", "ADE20KResNet18Layer2", "ADE20KResNet18Layer3", "ADE20KResNet18Layer4",
           "ADE20KResNet18Pyramid"]


class SynchronizedBatchNorm2d(nn.BatchNorm2d):
    """mit_semseg.lib.nn.SynchronizedBatchNorm2d on one device."""

    def __init__(self, num_features, eps=1e-5, momentum=0.001, affine=True):
        super().__init__(num_features, eps=eps, momentum=momentum, affine=affine)
        self.register_buffer('_tmp_running_mean', torch.zeros(self.num_features))
        self.register_buffer('_tmp_running_var', torch.ones(self.num_features))
        self.register_buffer('_running_iter', torch.ones(1))

    def forward(self, input):
        return F.batch_norm(input, self.running_mean, self.running_var, self.weight, self.bias, self.training,
                            self.momentum, self.eps)


def conv3x3(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = conv3x3(inplanes, planes, stride)
        self.bn1 = SynchronizedBatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = conv3x3(planes, planes)
        self.bn2 = SynchronizedBatchNorm2d(planes)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        residual = x
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        if self.downsample is not None:
            residual = self.downsample(x)
        return self.relu(out + residual)


class ResNet(nn.Module):
    """mit_semseg's resnet with the deep stem (conv1..bn3, maxpool) and layer1..layer4."""

    def __init__(self, block, layers):
        self.inplanes = 128
        super().__init__()
        self.conv1 = conv3x3(3, 64, stride=2)
        self.bn1 = SynchronizedBatchNorm2d(64)
        self.relu1 = nn.ReLU(inplace=True)
        self.conv2 = conv3x3(64, 64)
        self.bn2 = SynchronizedBatchNorm2d(64)
        self.relu2 = nn.ReLU(inplace=True)
        self.conv3 = conv3x3(64, 128)
        self.bn3 = SynchronizedBatchNorm2d(128)
        self.relu3 = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(block, 256, layers[2], stride=2)
        self.layer4 = self._make_layer(block, 512, layers[3], stride=2)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2. / n))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, planes * block.expansion, kernel_size=1, stride=stride, bias=False),
                SynchronizedBatchNorm2d(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes))
        return nn.Sequential(*layers)


class ResnetDilated(nn.Module):
    """mit_semseg's ResnetDilated(orig_resnet, dilate_scale=8): layer3 / layer4 lose their stride and dilate."""

    def __init__(self, orig_resnet, dilate_scale=8):
        super().__init__()
        from functools import partial
        orig_resnet.layer3.apply(partial(self._nostride_dilate, dilate=2))
        orig_resnet.layer4.apply(partial(self._nostride_dilate, dilate=4))
        for name in ["conv1", "bn1", "relu1", "conv2", "bn2", "relu2", "conv3", "bn3", "relu3", "maxpool",
                     "layer1", "layer2", "layer3", "layer4"]:
            setattr(self, name, getattr(orig_resnet, name))

    def _nostride_dilate(self, m, dilate):
        if m.__class__.__name__.find('Conv') != -1:
            if m.stride == (2, 2):
                m.stride = (1, 1)
                if m.kernel_size == (3, 3):
                    m.dilation = (dilate // 2, dilate // 2)
                    m.padding = (dilate // 2, dilate // 2)
            elif m.kernel_size == (3, 3):
                m.dilation = (dilate, dilate)
                m.padding = (dilate, dilate)


class ModelBuilder:
    @staticmethod
    def build_encoder(arch='resnet50dilated', fc_dim=512, weights=''):
        assert arch == 'resnet18dilated', arch
        net = ResnetDilated(ResNet(BasicBlock, [2, 2, 2, 2]), dilate_scale=8)
        if len(weights) > 0:
            net.load_state_dict(torch.load(weights, map_location='cpu'), strict=True)
        return net


def _cfg():
    def merge_from_file(path):
        assert os.path.basename(path) == "resnet18dilated-ppm_deepsup.yaml", path
        cfg.MODEL = types.SimpleNamespace(arch_encoder="resnet18dilated", fc_dim=512)
        cfg.TEST = types.SimpleNamespace(checkpoint="epoch_20.pth")
    cfg = types.SimpleNamespace(merge_from_file=merge_from_file)
    return cfg


def load_reference_image():
    """The reference's modalities/image.py, executed with the mit_semseg restatement above."""
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
    ref_loader._stub("mit_semseg.config").cfg = _cfg()
    ref_loader._stub("mit_semseg.models").ModelBuilder = ModelBuilder
    ref_loader._stub("mit_semseg.lib.nn").SynchronizedBatchNorm2d = SynchronizedBatchNorm2d
    return ref_loader._load(name, "torch_points3d/modules/multimodal/modalities/image.py")


def checkpoint_path(image):
    return os.path.join(image.PRETRAINED_DIR, "ade20k", "resnet18dilated-ppm_deepsup", "encoder_epoch_20.pth")


def make_keys(image):
    sd = torch.load(checkpoint_path(image), map_location="cpu")
    out = {"ckpt_keys": np.array(list(sd)), "ckpt_shapes": np.array([str(tuple(v.shape)) for v in sd.values()])}
    for cls in CLASSES:
        out[f"keys:{cls}"] = np.array(list(getattr(image, cls)().state_dict()))
    return out


def make_layer0(image):
    """The real layer0 slice, and an eval-mode and a train-mode TruncatedLayer0 step on it in float64."""
    ref = image.ADE20KResNet18TruncatedLayer0()
    out = {k: v.numpy() for k, v in ref.state_dict().items()}
    gen = torch.Generator().manual_seed(5)
    x = (torch.randint(-64, 65, (2, 3, 50, 66), generator=gen).double() / 32)
    gy = (torch.randint(-64, 65, (2, 128, 13, 17), generator=gen).double() / 32)
    out["x"], out["gy"] = x.numpy(), gy.numpy()
    for mode in ("eval", "train"):
        net = image.ADE20KResNet18TruncatedLayer0().double().train(mode == "train")
        xr = x.clone().requires_grad_(True)
        y = net(xr)
        params = list(net.parameters())
        g = torch.autograd.grad(y, [xr] + params, gy)
        out[f"{mode}:y"] = y.detach().float().numpy()
        out[f"{mode}:y_norm"] = np.float64(y.detach().norm())
        out[f"{mode}:gx_norm"] = np.float64(g[0].norm())
        for (k, _), gp in zip(net.named_parameters(), g[1:]):
            out[f"{mode}:gnorm:{k}"] = np.float64(gp.norm())
        for k, v in net.state_dict().items():
            if "running_" in k:
                out[f"{mode}:after:{k}"] = v.numpy()
    return out


# name -> (class, kwargs, training, input shape, seed): the BasicBlock layers with their downsamples, the dilated
# layer3 / layer4, a scale_factor resize and the Pyramid
CASES = {
    "tl4_train": ("ADE20KResNet18TruncatedLayer4", {}, True, (2, 3, 61, 45), 1),
    "layer3_train": ("ADE20KResNet18Layer3", {}, True, (2, 128, 13, 11), 2),
    "layer2_eval": ("ADE20KResNet18Layer2", {}, False, (1, 64, 15, 18), 3),
    "tl2_sf8_eval": ("ADE20KResNet18TruncatedLayer2", {"scale_factor": -1}, False, (2, 3, 21, 30), 4),
    "pyramid_sf2_train": ("ADE20KResNet18Pyramid", {"scale_factor": 2}, True, (2, 3, 24, 40), 5),
}


def case_inputs(net, shape, seed):
    """(state, x) of a case: hashed parameters and running stats, and a hashed input on a grid of 1/4."""
    state = O.hashed_state(net.state_dict(), seed)
    x = torch.from_numpy(O.hash_grid(seed, 50000, shape, 8, 2))
    return state, x


def case_upstream(shape, seed):
    return torch.from_numpy(O.hash_grid(seed, 60000, shape, 8, 3))


def make_case(image, cls, kwargs, training, shape, seed):
    net = getattr(image, cls)(**kwargs).double().train(training)
    state, x = case_inputs(net, shape, seed)
    net.load_state_dict(state, strict=True)
    x = x.clone().requires_grad_(True)
    y = net(x)
    gy = case_upstream(tuple(y.shape), seed)
    names = [k for k, _ in net.named_parameters()]
    g = torch.autograd.grad(y, [x] + list(net.parameters()), gy)
    out = {"y": y.detach().float().numpy(), "y_norm": np.float64(y.detach().norm()),
           "gx": g[0].float().numpy(), "gx_norm": np.float64(g[0].norm())}
    for tag, (k, gp) in enumerate(zip(names, g[1:])):
        out[f"gnorm:{k}"] = np.float64(gp.norm())
        out[f"gproj:{k}"] = np.float64((gp * O.projection(seed, tag, tuple(gp.shape))).sum())
    for k, v in net.state_dict().items():
        if k.endswith((".running_mean", ".running_var")):
            out[f"after:{k}"] = v.numpy()
        if k.endswith((".weight", ".bias", ".running_mean", ".running_var")):
            out[f"checksum:{k}"] = np.float64(state[k].double().sum())
    out["checksum:x"] = np.float64(x.detach().sum())
    return out


def main():
    os.environ.setdefault("PYTORCH_JIT", "0")
    image = load_reference_image()
    cases = [(name, make_case(image, *spec)) for name, spec in CASES.items()]
    for name, d in [("keys", make_keys(image)), ("layer0", make_layer0(image))] + cases:
        path = os.path.join(OUT, f"image_resnet18_{name}.npz")
        np.savez_compressed(path, **d)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
