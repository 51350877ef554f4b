"""Float64 restatement of the reference's ADE20KResNet18PPM (torch_points3d/modules/multimodal/modalities/
image.py:634-790): mit_semseg's resnet18dilated trunk (oracle/image_resnet18_oracle.py) and PPMFeatMap, in plain
torch on the CPU.

The head on conv5 [B, C, h, w]: for each pool scale s in (1, 2, 3, 6), F.adaptive_avg_pool2d to s x s, a 1x1 conv
without bias, BatchNorm (PrudentSynchronizedBatchNorm2d: eval mode for a (1, C, 1, 1) input, i.e. s = 1 at B = 1) and
ReLU, then F.interpolate back to (h, w) (bilinear, align_corners=False, size-based); conv5 and the four branches
concatenated, then conv_last = 3x3 conv (padding 1, no bias), BatchNorm and ReLU; an optional final resize to
out_size.  BatchNorm is F.batch_norm(training, momentum 0.001, eps 1e-5) and updates the buffers it is given.

`params` maps the module's state-dict keys (encoder.conv1.weight, ..., decoder.ppm.<i>.1.weight, ...,
decoder.conv_last.1.*) to tensors.  `masks`, when given, holds the branch decisions of another run in forward order:
those of the trunk (image_resnet18_oracle), then a 0/1 tensor per pyramid branch's ReLU and one for conv_last's."""
import torch
import torch.nn.functional as F

from oracle import image_resnet18_oracle as R

SCALES = (1, 2, 3, 6)
LAYERS = ["layer0", "layer1", "layer2", "layer3", "layer4"]
STEM = {"conv1": "0", "bn1": "1", "conv2": "3", "bn2": "4", "conv3": "6", "bn3": "7"}


def trunk_params(p):
    """The encoder.* entries of p under the keys image_resnet18_oracle reads (conv.<i>.*), the same tensors."""
    out = {}
    for k, v in p.items():
        if k.startswith("encoder."):
            head, rest = k[len("encoder."):].split(".", 1)
            out[f"conv.0.{STEM[head]}.{rest}" if head in STEM else f"conv.{int(head[5:])}.{rest}"] = v
    return out


def head(conv5, p, training, out_size=None, masks=None):
    """PPMFeatMap.forward on conv5 [B, C, h, w]."""
    B, _, h, w = conv5.shape
    outs = [conv5]
    for i, s in enumerate(SCALES):
        pre = f"decoder.ppm.{i}"
        v = F.conv2d(F.adaptive_avg_pool2d(conv5, s), p[pre + ".1.weight"])
        v = R._relu(R._bn(v, p, pre + ".2", training and not (B == 1 and s == 1)), masks)
        outs.append(F.interpolate(v, (h, w), mode="bilinear", align_corners=False))
    x = F.conv2d(torch.cat(outs, 1), p["decoder.conv_last.0.weight"], padding=1)
    x = R._relu(R._bn(x, p, "decoder.conv_last.1", training), masks)
    if out_size is not None:
        x = F.interpolate(x, size=tuple(out_size), mode="bilinear", align_corners=False)
    return x


def forward(x, p, training, out_size=None, masks=None):
    """ADE20KResNet18PPM.forward(x, out_size=out_size) with every BatchNorm in mode `training`."""
    it = None if masks is None else iter(masks)
    conv5 = R.trunk_layers(x, trunk_params(p), LAYERS, training, it)[-1]
    return head(conv5, p, training, out_size, it)
