"""Float64 torch restatement of the reference's image UNet (modalities/image.py:343-627), extending
image_encoder_oracle.py: ResNetUp stages of ConvTranspose2dWS (standardised per input channel, fan = C_out, zero
padding), GroupNorm and ReLUWS, transposed ResBlocks with a plain 1x1 nn.Conv2d downsample, the symmetric skip
stack, and UnaryConv with explicit dropout masks.  F.conv_transpose2d + F.conv2d + F.group_norm on the CPU (or any
device); parameters are read from a UNet state dict."""
import torch
import torch.nn.functional as F

from oracle import image_encoder_oracle as E


def convt_ws(x, w, b, stride, padding):
    # standardize_weights on a [C_in, C_out, R, S] weight: statistics over dim 0's filters, sqrt(weight.shape[1])
    return F.conv_transpose2d(x, E.standardize(w), b, stride=stride, padding=padding)


def res_block_t(x, sd, p):
    h = E.relu_ws(E.gn(convt_ws(x, sd[p + "block.0.weight"], sd[p + "block.0.bias"], 1, 1), sd, p + "block.1"))
    h = E.relu_ws(E.gn(convt_ws(h, sd[p + "block.3.weight"], sd[p + "block.3.bias"], 1, 1), sd, p + "block.4"))
    if p + "downsample.0.weight" in sd:
        skip = E.gn(F.conv2d(x, sd[p + "downsample.0.weight"], sd[p + "downsample.0.bias"]), sd, p + "downsample.1")
    else:
        skip = x
    return h + skip


def resnet_up(x, skip, sd, kernel_size, stride, padding, skip_first=False):
    """One ResNetUp stage; sd holds its state dict (conv_in.*, blocks.<i>.*)."""
    if skip_first and skip is not None:
        x = torch.cat((x, skip), dim=1)
    if "conv_in.0.weight" in sd:
        x = E.relu_ws(E.gn(convt_ws(x, sd["conv_in.0.weight"], sd["conv_in.0.bias"], stride, padding), sd,
                           "conv_in.1"))
    if not skip_first and skip is not None:
        x = torch.cat((x, skip), dim=1)
    i = 0
    while f"blocks.{i}.block.0.weight" in sd:
        x = res_block_t(x, sd, f"blocks.{i}.")
        i += 1
    return x


def unary_conv(x, sd, standardize=False, activation=None, in_mask=None, out_mask=None):
    """UnaryConv: x * in_mask -> 1x1 conv (standardised or not) -> relu (x ReLUWS scale when standardised) ->
    * out_mask; a mask is [B or 1, C, 1, 1] or None."""
    if in_mask is not None:
        x = x * in_mask
    w = sd["conv.weight"]
    x = F.conv2d(x, E.standardize(w) if standardize else w, sd["conv.bias"])
    if activation is not None:
        x = F.relu(x) * (E.RELU_WS_SCALE if standardize else 1.0)
    if out_mask is not None:
        x = x * out_mask
    return x


def sub(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def unet(x, sd, down, up, last=None, skip_first=False):
    """sd: a UNet state dict; down / up: [(kernel_size, stride, padding)] per stage; last: UnaryConv options
    (standardize, activation, in_mask, out_mask) as a dict, or None when there is no last_conv."""
    stack = []
    for i, shape in enumerate(down):
        x = E.resnet_down(x, sub(sd, f"down_modules.{i}."), *shape)
        stack.append(x)
    stack.pop(-1)
    if skip_first:
        stack.append(None)
    for i, shape in enumerate(up):
        skip = stack.pop(-1) if stack else None
        x = resnet_up(x, skip, sub(sd, f"up_modules.{i}."), *shape, skip_first=skip_first)
    if last is not None:
        x = unary_conv(x, sub(sd, "last."), **last)
    return x
