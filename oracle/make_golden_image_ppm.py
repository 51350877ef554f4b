"""Fixtures of ADE20KResNet18PPM, made by EXECUTING the reference's wrapper (torch_points3d/modules/multimodal/
modalities/image.py:634-790), loaded by file path in float64 on the CPU.

    PYTORCH_JIT=0 python -m oracle.make_golden_image_ppm      # writes tests/golden/image_ppm_*.npz

mit_semseg is stubbed as in oracle/make_golden_image_resnet18.py (imported), plus a restatement of what the wrapper
takes from mit_semseg's decoder side: PPMDeepsup (ppm, cbr_deepsup, conv_last with its Dropout2d and 150-class
classifier, conv_last_deepsup) and ModelBuilder.build_decoder, which loads the reference's decoder_epoch_20.pth with
strict=True -- proof that the restated tree is the checkpoint's.  The config stub also answers arch_decoder and
DATASET.num_class = 150.

Files:
  image_ppm_keys.npz    the decoder checkpoint's key names and shapes (no values) and the reference state-dict keys
                        of ADE20KResNet18PPM;
  image_ppm_<case>.npz  seeded cases (CASES), with the integer-hash parameters and inputs of
                        oracle/image_resnet18_oracle.py (per-tensor checksums stored) and the quantities of
                        make_golden_image_resnet18: the output and the input gradient rounded to float32 with their
                        float64 norms (eval_outsize stores every 32nd channel of its full-size output), the running
                        stats after the step, and per parameter the gradient norm and its projection on a fixed +-1
                        direction.
tests/test_image_ppm_oracle.py checks oracle/image_ppm_oracle.py against every fixture."""
import os
import types

import numpy as np
import torch
import torch.nn as nn

from oracle import image_resnet18_oracle as O
from oracle import make_golden_image_resnet18 as G

OUT = G.OUT
NUM_CLASS = 150

# name -> (training, input shape, out_size, seed): conv5 8 x 6 (the bins of scales 3 and 6 overlap along h); batch
# size 1, where the scale-1 branch runs in eval mode (Prudent); conv5 5 x 7 (h < 6: bins repeat) with a final resize
CASES = {
    "train_b2": (True, (2, 3, 61, 45), None, 21),
    "train_b1": (True, (1, 3, 50, 66), None, 22),
    "eval_outsize": (False, (2, 3, 40, 56), (40, 56), 23),
}
Y_CHANNEL_STEP = {"eval_outsize": 32}


def conv3x3_bn_relu(in_planes, out_planes, stride=1):
    return nn.Sequential(nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False),
                         G.SynchronizedBatchNorm2d(out_planes), nn.ReLU(inplace=True))


class PPMDeepsup(nn.Module):
    """mit_semseg's PPMDeepsup module tree (the wrapper only takes .ppm and .conv_last from it)."""

    def __init__(self, num_class=150, fc_dim=4096, use_softmax=False, pool_scales=(1, 2, 3, 6)):
        super().__init__()
        self.use_softmax = use_softmax
        self.ppm = nn.ModuleList([nn.Sequential(nn.AdaptiveAvgPool2d(scale),
                                                nn.Conv2d(fc_dim, 512, kernel_size=1, bias=False),
                                                G.SynchronizedBatchNorm2d(512), nn.ReLU(inplace=True))
                                  for scale in pool_scales])
        self.cbr_deepsup = conv3x3_bn_relu(fc_dim // 2, fc_dim // 4, 1)
        self.conv_last = nn.Sequential(
            nn.Conv2d(fc_dim + len(pool_scales) * 512, 512, kernel_size=3, padding=1, bias=False),
            G.SynchronizedBatchNorm2d(512), nn.ReLU(inplace=True), nn.Dropout2d(0.1),
            nn.Conv2d(512, num_class, kernel_size=1))
        self.conv_last_deepsup = nn.Conv2d(fc_dim // 4, num_class, 1, 1, 0)
        self.dropout_deepsup = nn.Dropout2d(0.1)


class ResnetDilated(G.ResnetDilated):
    """make_golden_image_resnet18's ResnetDilated with mit_semseg's forward."""

    def forward(self, x, return_feature_maps=False):
        conv_out = []
        x = self.relu1(self.bn1(self.conv1(x)))
        x = self.relu2(self.bn2(self.conv2(x)))
        x = self.relu3(self.bn3(self.conv3(x)))
        x = self.maxpool(x)
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            x = layer(x)
            conv_out.append(x)
        return conv_out if return_feature_maps else [x]


class ModelBuilder(G.ModelBuilder):
    @staticmethod
    def build_encoder(arch='resnet50dilated', fc_dim=512, weights=''):
        assert arch == 'resnet18dilated', arch
        net = ResnetDilated(G.ResNet(G.BasicBlock, [2, 2, 2, 2]), dilate_scale=8)
        if len(weights) > 0:
            net.load_state_dict(torch.load(weights, map_location='cpu'), strict=True)
        return net

    @staticmethod
    def weights_init(m):
        classname = m.__class__.__name__
        if classname.find('Conv') != -1:
            nn.init.kaiming_normal_(m.weight.data)
        elif classname.find('BatchNorm') != -1:
            m.weight.data.fill_(1.)
            m.bias.data.fill_(1e-4)

    @staticmethod
    def build_decoder(arch='ppm_deepsup', fc_dim=512, num_class=150, weights='', use_softmax=False):
        assert arch == 'ppm_deepsup', arch
        net = PPMDeepsup(num_class=num_class, fc_dim=fc_dim, use_softmax=use_softmax)
        net.apply(ModelBuilder.weights_init)
        if len(weights) > 0:
            net.load_state_dict(torch.load(weights, map_location='cpu'), strict=True)
        return net


def _cfg():
    def merge_from_file(path):
        assert os.path.basename(path) == "resnet18dilated-ppm_deepsup.yaml", path
        cfg.MODEL = types.SimpleNamespace(arch_encoder="resnet18dilated", arch_decoder="ppm_deepsup", fc_dim=512)
        cfg.DATASET = types.SimpleNamespace(num_class=NUM_CLASS)
        cfg.TEST = types.SimpleNamespace(checkpoint="epoch_20.pth")
    cfg = types.SimpleNamespace(merge_from_file=merge_from_file)
    return cfg


def load_reference_image():
    """The reference's modalities/image.py with the encoder stub of make_golden_image_resnet18 and the decoder side
    above."""
    image = G.load_reference_image()
    image.MITCfg = _cfg()
    image.MITModelBuilder = ModelBuilder
    return image


def checkpoint_dir(image):
    return os.path.join(image.PRETRAINED_DIR, "ade20k", "resnet18dilated-ppm_deepsup")


def make_keys(image):
    sd = torch.load(os.path.join(checkpoint_dir(image), "decoder_epoch_20.pth"), map_location="cpu")
    return {"ckpt_keys": np.array(list(sd)), "ckpt_shapes": np.array([str(tuple(v.shape)) for v in sd.values()]),
            "keys:ADE20KResNet18PPM": np.array(list(image.ADE20KResNet18PPM().state_dict()))}


def case_inputs(net, shape, seed):
    return G.case_inputs(net, shape, seed)


def make_case(image, name, training, shape, out_size, seed):
    net = image.ADE20KResNet18PPM().double().train(training)
    state, x = case_inputs(net, shape, seed)
    net.load_state_dict(state, strict=True)
    x = x.clone().requires_grad_(True)
    y = net(x, out_size=out_size)
    gy = G.case_upstream(tuple(y.shape), seed)
    names = [k for k, _ in net.named_parameters()]
    g = torch.autograd.grad(y, [x] + list(net.parameters()), gy)
    step = Y_CHANNEL_STEP.get(name, 1)
    out = {"y": y.detach()[:, ::step].float().numpy(), "y_norm": np.float64(y.detach().norm()),
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
    cases = [(name, make_case(image, name, *spec)) for name, spec in CASES.items()]
    for name, d in [("keys", make_keys(image))] + cases:
        path = os.path.join(OUT, f"image_ppm_{name}.npz")
        np.savez_compressed(path, **d)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
