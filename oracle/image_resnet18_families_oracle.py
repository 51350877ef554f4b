"""Float64 restatement of the reference's ImageNet ResNet18* wrappers (torchvision's resnet18, torch_points3d/modules/
multimodal/modalities/image.py:959-1126) and Cityscapes CityscapesResNet18* wrappers (SFSegNets' ResNet-18,
image.py:1129-1399), in plain torch on the CPU.

The trunks: ImageNet layer0 = 7x7/2 conv (padding 3), BatchNorm, ReLU, MaxPool2d(3, 2, 1); Cityscapes layer0 =
3x3/2 conv, BN, ReLU, 3x3 conv, BN, ReLU, 3x3 conv (64 -> 128), BN, ReLU, MaxPool2d(3, 2, 0).  layer1..layer4 = two
BasicBlocks each, layer2..layer4 with stride 2, no dilation; the first block has a 1x1 downsample where the stride or
the width changes (Cityscapes layer1: 128 -> 64 at stride 1).  BatchNorm is nn.BatchNorm2d's: in training mode
num_batches_tracked += 1, then F.batch_norm(..., training, momentum, eps=1e-5) with momentum 0.1 (None: 1 /
num_batches_tracked), updating the running buffers it is given in place.

`params` maps the module's state-dict keys to tensors; `prefixes` gives each layer's key prefix (conv.<i> for the
wrappers, the layer name for CityscapesResNet18).  `masks`, when given, are another run's branch decisions in forward
order, as in oracle/image_resnet18_oracle.py: a 0/1 tensor per ReLU and the flat max index per max-pool window."""
import torch
import torch.nn.functional as F

from oracle.image_resnet18_oracle import hash_grid, hashed_state, projection  # noqa: F401  (the seeded parameters)

EPS = 1e-5
STRIDE = {"layer1": 1, "layer2": 2, "layer3": 2, "layer4": 2}
SCALE = {"layer0": 4, "layer1": 1, "layer2": 2, "layer3": 2, "layer4": 2}
# (conv key, BatchNorm key, stride) of each stem unit, and the max pool's padding
STEM = {"imagenet": ([("0", "1", 2)], 1),
        "cityscapes": ([("0.0", "0.1", 2), ("0.3", "0.4", 1), ("0.6", "1", 1)], 0)}


def _bn(x, p, key, training, momentum):
    if training:
        p[key + ".num_batches_tracked"] += 1
        if momentum is None:
            momentum = 1.0 / float(p[key + ".num_batches_tracked"])
    return F.batch_norm(x, p[key + ".running_mean"], p[key + ".running_var"], p[key + ".weight"], p[key + ".bias"],
                        training, 0.0 if momentum is None else momentum, EPS)


def _conv(x, w, stride=1):
    return F.conv2d(x, w, stride=stride, padding=(w.shape[-1] - 1) // 2)


def _relu(v, masks):
    return F.relu(v) if masks is None else v * next(masks).to(v)


def _pool(x, padding, masks):
    if masks is None:
        return F.max_pool2d(x, 3, 2, padding)
    idx = next(masks).to(x.device)
    B, C, Ho, Wo = idx.shape
    return x.flatten(2).gather(2, idx.flatten(2)).view(B, C, Ho, Wo)


def layer0(x, p, pre, family, training, momentum=0.1, masks=None):
    units, padding = STEM[family]
    for conv, bn, stride in units:
        x = _relu(_bn(_conv(x, p[f"{pre}.{conv}.weight"], stride), p, f"{pre}.{bn}", training, momentum), masks)
    return _pool(x, padding, masks)


def basic_block(x, p, pre, stride, training, momentum=0.1, masks=None):
    h = _relu(_bn(_conv(x, p[f"{pre}.conv1.weight"], stride), p, f"{pre}.bn1", training, momentum), masks)
    out = _bn(_conv(h, p[f"{pre}.conv2.weight"]), p, f"{pre}.bn2", training, momentum)
    if f"{pre}.downsample.0.weight" in p:
        res = _bn(_conv(x, p[f"{pre}.downsample.0.weight"], stride), p, f"{pre}.downsample.1", training, momentum)
    else:
        res = x
    return _relu(out + res, masks)


def trunk_layers(x, p, family, layers, training, momentum=0.1, masks=None, prefixes=None):
    """The output of every layer of `layers`, in order."""
    prefixes = prefixes or [f"conv.{i}" for i in range(len(layers))]
    outs = []
    for pre, name in zip(prefixes, layers):
        if name == "layer0":
            x = layer0(x, p, pre, family, training, momentum, masks)
        else:
            x = basic_block(x, p, f"{pre}.0", STRIDE[name], training, momentum, masks)
            x = basic_block(x, p, f"{pre}.1", 1, training, momentum, masks)
        outs.append(x)
    return outs


def conv_scale_factor(layers):
    s = 1
    for name in layers:
        s *= SCALE[name]
    return s


def forward(x, p, family, layers, training, scale_factor=None, pyramid=False, momentum=0.1, masks=None,
            prefixes=None):
    """The wrappers' forward (scale_factor < 0 already replaced by conv_scale_factor), or the Pyramid's when
    pyramid=True; CityscapesResNet18 is layers = all five with prefixes = their names."""
    outs = trunk_layers(x, p, family, layers, training, momentum, None if masks is None else iter(masks), prefixes)
    if pyramid:
        size = [int(s * scale_factor / conv_scale_factor(layers)) for s in x.shape[2:4]]
        return torch.cat([F.interpolate(o, size=size, mode="bilinear", align_corners=False) for o in outs], dim=1)
    y = outs[-1]
    if scale_factor is not None:
        y = F.interpolate(y, scale_factor=scale_factor, mode="bilinear", align_corners=False)
    return y
