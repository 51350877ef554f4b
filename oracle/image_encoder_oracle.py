"""Float64 torch restatement of the reference's from-scratch image encoder (modalities/image.py:39-340):
ResNetDown stages of Conv2dWS (weight standardisation: unbiased std + 1e-5, fan_in = C_in, sqrt in float32), GroupNorm, ReLUWS and
ResBlocks whose residual is added after the second activation.  F.pad(reflect) + F.conv2d + F.group_norm on the CPU
(or any device); the stage parameters are read from a ResNetDown state dict."""
import math

import torch
import torch.nn.functional as F

RELU_WS_SCALE = math.sqrt(2 / (1 - 1 / math.pi))


def standardize(w):
    w = w - w.mean(dim=(1, 2, 3), keepdim=True)
    std = w.reshape(w.shape[0], -1).std(dim=1).reshape(-1, 1, 1, 1) + 1e-5
    # fan_in is torch.Tensor([C_in]): its square root is taken in float32 (image.py:44-47)
    return w / (std * float(torch.sqrt(torch.tensor([float(w.shape[1])], dtype=torch.float32))))


def conv_ws(x, w, b, stride, padding):
    if padding:
        x = F.pad(x, (padding,) * 4, mode="reflect")
    return F.conv2d(x, standardize(w), b, stride=stride)


def gn(x, sd, prefix, eps=1e-5):
    g = sd[prefix + ".weight"]
    return F.group_norm(x, max(g.numel() // 16, 1), g, sd[prefix + ".bias"], eps)


def relu_ws(x):
    return F.relu(x) * RELU_WS_SCALE


def res_block(x, sd, p):
    h = relu_ws(gn(conv_ws(x, sd[p + "block.0.weight"], sd[p + "block.0.bias"], 1, 1), sd, p + "block.1"))
    h = relu_ws(gn(conv_ws(h, sd[p + "block.3.weight"], sd[p + "block.3.bias"], 1, 1), sd, p + "block.4"))
    if p + "downsample.0.weight" in sd:
        skip = gn(F.conv2d(x, sd[p + "downsample.0.weight"], sd[p + "downsample.0.bias"]), sd, p + "downsample.1")
    else:
        skip = x
    return h + skip


def resnet_down(x, sd, kernel_size, stride, padding):
    """One ResNetDown stage; sd holds its state dict (conv_in.*, blocks.<i>.*)."""
    if "conv_in.0.weight" not in sd:
        return x
    x = relu_ws(gn(conv_ws(x, sd["conv_in.0.weight"], sd["conv_in.0.bias"], stride, padding), sd, "conv_in.1"))
    i = 0
    while f"blocks.{i}.block.0.weight" in sd:
        x = res_block(x, sd, f"blocks.{i}.")
        i += 1
    return x


def encoder(x, stages):
    """stages: [(state dict, kernel_size, stride, padding)] applied in order."""
    for sd, k, s, p in stages:
        x = resnet_down(x, sd, k, s, p)
    return x
