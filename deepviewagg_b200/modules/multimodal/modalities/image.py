"""The from-scratch image encoder of the reference (torch_points3d/modules/multimodal/modalities/image.py:26-340):
ResNetDown built from ResBlock, Conv2dWS, GroupNorm and ReLUWS, with the reference's names, constructor arguments
and module tree, so a reference state_dict loads with strict=True.

ResNetDown.forward and ResBlock.forward run on the sm_90a kernels of libdva_conv2d.so (ops.conv_gn_relu_ws,
ops.res_block): each Conv2dWS -> GroupNorm -> ReLUWS unit, and each ResBlock, is one autograd node; Conv2dWS,
GroupNorm and ReLUWS only hold the parameters.  Input [B, C, H, W] on CUDA, NCHW or channels-last; the kernels
compute from fp32 operands whatever the dtype of the input and the parameters (a half or double input is cast), and
the output, the reference's shape and values with channels-last strides, is in the input's dtype (fp32 under
autocast).

Supported: block='ResBlock', normalization='GroupNorm', weight_standardization=True, padding_mode='reflect',
dilation=1, and (kernel_size, stride, padding) of conv_in in {(3, 1, 1), (2, 2, 0)} -- every layer of the shipped
GroupNorm configs.  Anything else raises NotImplementedError naming the argument.
"""
from math import pi, sqrt

import torch
import torch.nn as nn

from .... import ops
from ...._lib import require_cuda
from ....core.common_modules import Identity


class Seq(nn.Sequential):
    """nn.Sequential whose children are named '0', '1', ... in append order (base_modules.py:159-167)."""

    def __init__(self):
        super().__init__()
        self._num_modules = 0

    def append(self, module):
        self.add_module(str(self._num_modules), module)
        self._num_modules += 1
        return self


class ModalityIdentity(Identity):
    """Identity that swallows extra constructor and forward arguments (image.py:26-36)."""

    def __init__(self, **kwargs):
        super().__init__()

    def forward(self, x, *args, **kwargs):
        return x


def standardize_weights(weight, scaled=True):
    """Weight standardisation of image.py:39-50, in torch: unbiased std + 1e-5, fan_in = weight.shape[1]."""
    weight_mean = weight.mean(dim=1, keepdim=True).mean(dim=2, keepdim=True).mean(dim=3, keepdim=True)
    weight = weight - weight_mean
    std = weight.view(weight.size(0), -1).std(dim=1).view(-1, 1, 1, 1) + 1e-5
    # torch.Tensor([C_in]) in the reference: the square root is taken in float32 whatever the weights' dtype
    fan_in = torch.tensor([float(weight.shape[1])], dtype=torch.float32, device=weight.device)
    if scaled:
        return weight / (std.expand_as(weight) * torch.sqrt(fan_in))
    return weight / std.expand_as(weight)


class Conv2dWS(nn.Conv2d):
    """Parameters of a weight-standardised convolution (image.py:53-73).  It runs inside ResNetDown / ResBlock."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True,
                 padding_mode='zeros', scaled=True):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                         groups=groups, bias=bias, padding_mode=padding_mode)
        self.scaled = scaled

    def forward(self, x, *args, **kwargs):
        raise NotImplementedError("Conv2dWS runs fused with its GroupNorm and ReLUWS: call the ResNetDown or "
                                  "ResBlock that holds it")


class ReLUWS(nn.ReLU):
    """relu(x) * sqrt(2 / (1 - 1/pi)) (image.py:110-125); fused into the GroupNorm pass of ResNetDown / ResBlock."""
    _SCALE = sqrt(2 / (1 - 1 / pi))

    def forward(self, input, *args, **kwargs):
        raise NotImplementedError("ReLUWS runs fused with its convolution and GroupNorm: call the ResNetDown or "
                                  "ResBlock that holds it")

    def extra_repr(self) -> str:
        return f"inplace={self.inplace}"


def _group_norm(nc):
    # ~16 channels per group (image.py:296-297)
    return nn.GroupNorm(max(nc // 16, 1), nc)


def _rows(x):
    """[B, C, H, W] CUDA (any memory format) -> channels-last rows [B, H, W, C], contiguous (the operators cast
    them to fp32)."""
    require_cuda(x)
    if x.dim() != 4:
        raise ValueError(f"expected a [B, C, H, W] image batch, got shape {tuple(x.shape)}")
    if not x.is_floating_point():
        raise TypeError(f"expected a floating-point image batch, got {x.dtype}")
    return x.permute(0, 2, 3, 1).contiguous()


def _out_dtype(x):
    # the dtype of the input, as the reference's layers give; under autocast the fp32 result (ops.linear's rule)
    return torch.float32 if torch.is_autocast_enabled("cuda") else x.dtype


class ResBlock(nn.Module):
    """Basic ResNet block (image.py:128-189): conv3x3-GN-ReLUWS-conv3x3-GN-ReLUWS, plus the block input or a 1x1
    nn.Conv2d + GN downsample when the widths differ, added after the second activation."""

    def __init__(self, input_nc, output_nc, convolution, normalization, activation):
        super().__init__()
        if convolution is not Conv2dWS:
            raise NotImplementedError(f"convolution={getattr(convolution, '__name__', convolution)}: only Conv2dWS")
        if activation is not ReLUWS:
            raise NotImplementedError(f"activation={getattr(activation, '__name__', activation)}: only ReLUWS")
        self.block = (
            Seq().append(convolution(input_nc, output_nc, kernel_size=3, stride=1, padding=1, padding_mode='reflect'))
            .append(normalization(output_nc))
            .append(activation())
            .append(convolution(output_nc, output_nc, kernel_size=3, stride=1, padding=1, padding_mode='reflect'))
            .append(normalization(output_nc))
            .append(activation()))
        if not isinstance(self.block[1], nn.GroupNorm):
            raise NotImplementedError("normalization: only nn.GroupNorm")
        if input_nc != output_nc:
            self.downsample = (
                Seq().append(nn.Conv2d(input_nc, output_nc, kernel_size=1, stride=1))
                .append(normalization(output_nc)))
        else:
            self.downsample = None

    def forward_rows(self, x):
        """The block on channels-last rows [B, H, W, C_in] -> [B, H, W, C_out]."""
        ops.conv_out_hw(ops.CONV_KINDS[(3, 1, 1)], x.shape[1], x.shape[2])
        return ops.res_block(x, self)

    def forward(self, x, *args, **kwargs):
        return self.forward_rows(_rows(x)).to(_out_dtype(x)).permute(0, 3, 1, 2)


def _is_list(x):
    return isinstance(x, (list, tuple)) or type(x).__name__ == "ListConfig"


def _single(v, name):
    if isinstance(v, (list, tuple)):
        if len(set(v)) != 1:
            raise NotImplementedError(f"{name}={v}: only square kernels, strides and paddings")
        v = v[0]
    return int(v)


class ResNetDown(nn.Module):
    """in -- strided conv -- N x ResBlock (image.py:251-340), on the sm_90a kernels of libdva_conv2d.so."""

    CONVOLUTION = "Conv2d"
    ACTIVATION = "ReLU"

    def __init__(self, down_conv_nn=[], kernel_size=2, dilation=1, stride=2, N=1, padding=0, block="ResBlock",
                 padding_mode='reflect', normalization='BatchNorm2d', weight_standardization=False, **kwargs):
        super().__init__()
        # an empty down_conv_nn or a negative width: pass-through (image.py:270-276)
        if len(down_conv_nn) < 2 or any([x < 0 for x in down_conv_nn]):
            self.conv_in = None
            self.blocks = None
            return
        if block != "ResBlock":
            raise NotImplementedError(f"block={block!r}: only 'ResBlock' is supported")
        if normalization != "GroupNorm":
            raise NotImplementedError(f"normalization={normalization!r}: only 'GroupNorm' is supported")
        if not weight_standardization:
            raise NotImplementedError("weight_standardization=False: only weight-standardised convolutions are "
                                      "supported")
        if padding_mode != "reflect":
            raise NotImplementedError(f"padding_mode={padding_mode!r}: only 'reflect' is supported")
        if _single(dilation, "dilation") != 1:
            raise NotImplementedError(f"dilation={dilation}: only 1 is supported")
        shape = (_single(kernel_size, "kernel_size"), _single(stride, "stride"), _single(padding, "padding"))
        if shape not in ((3, 1, 1), (2, 2, 0)):
            raise NotImplementedError(f"(kernel_size, stride, padding)={shape}: only (3, 1, 1) and (2, 2, 0) are "
                                      f"supported")
        self._kind = ops.CONV_KINDS[shape]

        nc_in, nc_stride_out, nc_block_in, nc_out = self._parse_conv_nn(down_conv_nn, stride, N)
        self.conv_in = (
            Seq().append(Conv2dWS(in_channels=nc_in, out_channels=nc_stride_out, kernel_size=kernel_size,
                                  stride=stride, dilation=dilation, padding=padding, padding_mode=padding_mode))
            .append(_group_norm(nc_stride_out))
            .append(ReLUWS()))
        if N > 0:
            self.blocks = Seq()
            for _ in range(N):
                self.blocks.append(ResBlock(nc_block_in, nc_out, Conv2dWS, _group_norm, ReLUWS))
                nc_block_in = nc_out
        else:
            self.blocks = None

    def _parse_conv_nn(self, down_conv_nn, stride, N):
        if _is_list(down_conv_nn[0]):
            down_conv_nn = down_conv_nn[0]
        assert len(down_conv_nn) == 2, \
            f"ResNetDown expects down_conv_nn to have length of 2 to carry (nc_in, nc_out) but got " \
            f"len(down_conv_nn)={len(down_conv_nn)}."
        nc_in, nc_out = down_conv_nn
        nc_stride_out = nc_in if _single(stride, "stride") > 1 and N > 0 else nc_out
        return nc_in, nc_stride_out, nc_stride_out, nc_out

    def output_hw(self, H, W):
        """Spatial size of the output for an H x W input; ValueError where the reference's padding or conv raises."""
        if self.conv_in is None:
            return H, W
        H, W = ops.conv_out_hw(self._kind, H, W)
        if self.blocks is not None:
            ops.conv_out_hw(ops.CONV_KINDS[(3, 1, 1)], H, W)
        return H, W

    def forward(self, x, *args, **kwargs):
        if self.conv_in is None:
            return x
        h = _rows(x)
        self.output_hw(h.shape[1], h.shape[2])
        conv, norm, _ = self.conv_in
        h = ops.conv_gn_relu_ws(h, conv, norm, self._kind)
        if self.blocks is not None:
            for blk in self.blocks:
                h = ops.res_block(h, blk)
        return h.to(_out_dtype(x)).permute(0, 3, 1, 2)
