"""Float64 restatement of the reference's ADE20KResNet18* wrappers (torch_points3d/modules/multimodal/modalities/
image.py:793-956) over mit_semseg's resnet18dilated trunk, in plain torch on the CPU.

The trunk: layer0 = 3 x (3x3 conv without bias, BatchNorm, ReLU) with the first convolution of stride 2, then
MaxPool2d(3, 2, 1); layer1..layer4 = two BasicBlocks each, layer2 with stride 2, layer3 / layer4 dilated (block-0
conv1 dilation 1 / 2, every other 3x3 2 / 4).  BatchNorm is F.batch_norm(x, running_mean, running_var, weight, bias,
training, momentum=0.001, eps=1e-5) and updates the running buffers it is given in place.

`params` maps the wrapper's state-dict keys (conv.<i>.*) to tensors; `layers` is the wrapper's _LAYERS.

`masks`, when given, holds the branch decisions of another run of the same network, in forward order: a 0/1 tensor
per ReLU (the stem units, then per BasicBlock its hidden and its output ReLU) and, for the max pool, the flat index of
each window's max (torch's max_pool2d indices).  The restatement then takes those branches instead of its own, so it
computes the same piecewise-linear function as that run."""
import math

import numpy as np
import torch
import torch.nn.functional as F

MOMENTUM, EPS = 0.001, 1e-5
LAYER_CFG = {  # name -> (stride of block 0, dilation of block-0 conv1, dilation of every other 3x3)
    "layer1": (1, 1, 1), "layer2": (2, 1, 1), "layer3": (1, 1, 2), "layer4": (1, 2, 4)}
SCALE = {"layer0": 4, "layer1": 1, "layer2": 2, "layer3": 1, "layer4": 1}


def _bn(x, p, key, training):
    return F.batch_norm(x, p[key + ".running_mean"], p[key + ".running_var"], p[key + ".weight"], p[key + ".bias"],
                        training, MOMENTUM, EPS)


def _conv(x, w, stride=1, dilation=1):
    pad = dilation if w.shape[-1] == 3 else 0
    return F.conv2d(x, w, stride=stride, padding=pad, dilation=dilation)


def _relu(v, masks):
    return F.relu(v) if masks is None else v * next(masks).to(v)


def _pool(x, masks):
    if masks is None:
        return F.max_pool2d(x, 3, 2, 1)
    idx = next(masks).to(x.device)
    B, C, Ho, Wo = idx.shape
    return x.flatten(2).gather(2, idx.flatten(2)).view(B, C, Ho, Wo)


def layer0(x, p, pre, training, masks=None):
    for conv, bn, stride in (("0", "1", 2), ("3", "4", 1), ("6", "7", 1)):
        x = _relu(_bn(_conv(x, p[f"{pre}.{conv}.weight"], stride), p, f"{pre}.{bn}", training), masks)
    return _pool(x, masks)


def basic_block(x, p, pre, stride, d1, d2, training, masks=None):
    h = _relu(_bn(_conv(x, p[f"{pre}.conv1.weight"], stride, d1), p, f"{pre}.bn1", training), masks)
    out = _bn(_conv(h, p[f"{pre}.conv2.weight"], 1, d2), p, f"{pre}.bn2", training)
    if f"{pre}.downsample.0.weight" in p:
        res = _bn(_conv(x, p[f"{pre}.downsample.0.weight"], stride), p, f"{pre}.downsample.1", training)
    else:
        res = x
    return _relu(out + res, masks)


def trunk_layers(x, p, layers, training, masks=None):
    """The output of every layer of `layers`, in order."""
    outs = []
    for i, name in enumerate(layers):
        if name == "layer0":
            x = layer0(x, p, f"conv.{i}", training, masks)
        else:
            stride, d0, d = LAYER_CFG[name]
            x = basic_block(x, p, f"conv.{i}.0", stride, d0, d, training, masks)
            x = basic_block(x, p, f"conv.{i}.1", 1, d, d, training, masks)
        outs.append(x)
    return outs


def conv_scale_factor(layers):
    s = 1
    for name in layers:
        s *= SCALE[name]
    return s


def forward(x, p, layers, training, scale_factor=None, pyramid=False, masks=None):
    """ADE20KResNet18TruncatedLayer4-style forward (scale_factor < 0 already replaced by conv_scale_factor), or the
    Pyramid's when pyramid=True."""
    outs = trunk_layers(x, p, layers, training, None if masks is None else iter(masks))
    if pyramid:
        size = [int(s * scale_factor / conv_scale_factor(layers)) for s in x.shape[2:4]]
        return torch.cat([F.interpolate(o, size=size, mode="bilinear", align_corners=False) for o in outs], dim=1)
    y = outs[-1]
    if scale_factor is not None:
        y = F.interpolate(y, scale_factor=scale_factor, mode="bilinear", align_corners=False)
    return y


# ---- seeded integer-hash parameters on a coarse binary grid (independent of torch's RNG): every value is m * 2^-e
# with a small integer m, so float32 holds it exactly and the fixtures need not store 11.3 M parameters
_M64 = (1 << 64) - 1


def _splitmix64(z):
    z = (z + np.uint64(0x9E3779B97F4A7C15)) & np.uint64(_M64)
    z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & np.uint64(_M64)
    z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & np.uint64(_M64)
    return z ^ (z >> np.uint64(31))


def hash_grid(seed, tag, shape, amp, exp):
    """float64 array of `shape`: (h mod (2 amp + 1) - amp) * 2^-exp, h the splitmix64 hash of (seed, tag, index)."""
    n = int(np.prod(shape)) if len(shape) else 1
    with np.errstate(over="ignore"):
        base = np.uint64((seed * 1000003 + tag * 7919) & _M64)
        h = _splitmix64(np.arange(n, dtype=np.uint64) + _splitmix64(base))
    m = (h >> np.uint64(33)) % np.uint64(2 * amp + 1)
    return ((m.astype(np.int64) - amp).astype(np.float64) * 2.0 ** -exp).reshape(shape)


def hashed_state(state_dict, seed):
    """Parameters and running stats for a wrapper state dict (its keys and shapes): conv weights near mit_semseg's
    std sqrt(2 / (k^2 C_out)), BN weight 1 +- 3/16, bias and running_mean +- 3/16, running_var 1 +- 3/8; the other
    buffers as they are.  Returns float64 tensors keyed like state_dict."""
    out = {}
    for tag, (k, v) in enumerate(state_dict.items()):
        shape = tuple(v.shape)
        if k.endswith(".weight") and v.dim() == 4:
            std = math.sqrt(2.0 / (shape[2] * shape[3] * shape[0]))
            exp = int(round(math.log2(math.sqrt(20.0 / 3.0) / std)))     # amp 4: std of m is sqrt(20/3) ~ 2.6
            a = hash_grid(seed, tag, shape, 4, exp)
        elif k.endswith(".weight"):
            a = 1 + hash_grid(seed, tag, shape, 3, 4)
        elif k.endswith(".bias") or k.endswith(".running_mean"):
            a = hash_grid(seed, tag, shape, 3, 4)
        elif k.endswith(".running_var"):
            a = 1 + hash_grid(seed, tag, shape, 3, 3)
        else:
            out[k] = v.detach().clone()
            continue
        out[k] = torch.from_numpy(a)
    return out


def projection(seed, tag, shape):
    """A fixed +-1 direction for the gradient projections of the fixtures."""
    return torch.from_numpy(np.where(hash_grid(seed, 100000 + tag, shape, 1, 0) > 0, 1.0, -1.0))
