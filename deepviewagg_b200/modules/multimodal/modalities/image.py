"""The from-scratch image network of the reference (torch_points3d/modules/multimodal/modalities/image.py:26-627):
the encoder ResNetDown built from ResBlock, Conv2dWS, GroupNorm and ReLUWS, and the decoder (ResNetUp,
ConvTranspose2dWS, UnaryConv, Dropout2d, PersistentDropout2d) that UNet joins to it, with the reference's names,
constructor arguments and module tree, so a reference state_dict loads with strict=True.

ResNetDown.forward and ResBlock.forward run on the sm_90a kernels of libdva_conv2d.so (ops.conv_gn_relu_ws,
ops.res_block): each Conv2dWS -> GroupNorm -> ReLUWS unit, and each ResBlock, is one autograd node; Conv2dWS,
GroupNorm and ReLUWS only hold the parameters.  Input [B, C, H, W] on CUDA, NCHW or channels-last; the kernels
compute from fp32 operands whatever the dtype of the input and the parameters (a half or double input is cast), and
the output, the reference's shape and values with channels-last strides, is in the input's dtype (fp32 under
autocast).

Supported: block='ResBlock', normalization='GroupNorm', weight_standardization=True, padding_mode='reflect',
dilation=1, and (kernel_size, stride, padding) of conv_in in {(3, 1, 1), (2, 2, 0)} -- every layer of the shipped
GroupNorm configs.  Anything else raises NotImplementedError naming the argument.

The decoder runs on the transposed convolutions of libdva_unet.so (ops.convt_gn_relu_ws, ops.res_block_t) with the
same rules; ResNetUp takes padding_mode='zeros' and (kernel_size, stride, padding) in {(2, 2, 0), (3, 1, 1)}, and
UnaryConv normalization=None.  UNet(opt) builds the network from the compact config format of the reference.
"""
from math import pi, sqrt

import torch
import torch.nn as nn
import torch.nn.functional as F

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


class ConvTranspose2dWS(nn.ConvTranspose2d):
    """Parameters of a weight-standardised transposed convolution (image.py:76-107); the weight is [C_in, C_out, R,
    S] and is standardised per input channel.  It runs inside ResNetUp / ResBlock."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, output_padding=0, dilation=1,
                 groups=1, bias=True, padding_mode='zeros', scaled=True):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=padding,
                         output_padding=output_padding, dilation=dilation, groups=groups, bias=bias,
                         padding_mode=padding_mode)
        self.scaled = scaled

    def forward(self, x, *args, output_size=None, **kwargs):
        raise NotImplementedError("ConvTranspose2dWS runs fused with its GroupNorm and ReLUWS: call the ResNetUp or "
                                  "ResBlock that holds it")


class ResBlock(nn.Module):
    """Basic ResNet block (image.py:128-189): conv3x3-GN-ReLUWS-conv3x3-GN-ReLUWS, plus the block input or a 1x1
    nn.Conv2d + GN downsample when the widths differ, added after the second activation.  The convolutions are
    Conv2dWS with reflect padding (the encoder) or ConvTranspose2dWS with zero padding (the decoder)."""

    def __init__(self, input_nc, output_nc, convolution, normalization, activation):
        super().__init__()
        if convolution is not Conv2dWS and convolution is not ConvTranspose2dWS:
            raise NotImplementedError(f"convolution={getattr(convolution, '__name__', convolution)}: only Conv2dWS "
                                      f"and ConvTranspose2dWS")
        if activation is not ReLUWS:
            raise NotImplementedError(f"activation={getattr(activation, '__name__', activation)}: only ReLUWS")
        self._transposed = convolution is ConvTranspose2dWS
        padding_mode = 'zeros' if self._transposed else 'reflect'
        self.block = (
            Seq().append(convolution(input_nc, output_nc, kernel_size=3, stride=1, padding=1, padding_mode=padding_mode))
            .append(normalization(output_nc))
            .append(activation())
            .append(convolution(output_nc, output_nc, kernel_size=3, stride=1, padding=1, padding_mode=padding_mode))
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
        if self._transposed:
            return ops.res_block_t(x, self)
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


class ResNetUp(ResNetDown):
    """in -- strided transposed conv -- [concatenate skip] -- N x ResBlock (image.py:343-405), the decoder stage, on
    the sm_90a kernels of libdva_unet.so.  skip_first=True concatenates the skip before the strided convolution."""

    CONVOLUTION = "ConvTranspose2d"

    def __init__(self, up_conv_nn=[], kernel_size=2, dilation=1, stride=2, N=1, padding=0, padding_mode='zeros',
                 normalization='BatchNorm2d', weight_standardization=False, skip_first=False, block="ResBlock",
                 **kwargs):
        nn.Module.__init__(self)
        self.skip_first = skip_first
        if len(up_conv_nn) < 2 or any([x < 0 for x in up_conv_nn]):
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
        if padding_mode != "zeros":
            raise NotImplementedError(f"padding_mode={padding_mode!r}: only 'zeros' is supported")
        if _single(dilation, "dilation") != 1:
            raise NotImplementedError(f"dilation={dilation}: only 1 is supported")
        shape = (_single(kernel_size, "kernel_size"), _single(stride, "stride"), _single(padding, "padding"))
        if shape not in ops.CONVT_KINDS:
            raise NotImplementedError(f"(kernel_size, stride, padding)={shape}: only (2, 2, 0) and (3, 1, 1) are "
                                      f"supported")
        if N < 0:
            raise NotImplementedError(f"N={N}: only N >= 0 is supported")
        self._kind = ops.CONVT_KINDS[shape]

        nc_in, nc_stride_out, nc_block_in, nc_out = self._parse_conv_nn(up_conv_nn, stride, N)
        self.conv_in = (
            Seq().append(ConvTranspose2dWS(in_channels=nc_in, out_channels=nc_stride_out, kernel_size=kernel_size,
                                           stride=stride, dilation=dilation, padding=padding,
                                           padding_mode=padding_mode))
            .append(_group_norm(nc_stride_out))
            .append(ReLUWS()))
        if N > 0:
            self.blocks = Seq()
            for _ in range(N):
                self.blocks.append(ResBlock(nc_block_in, nc_out, ConvTranspose2dWS, _group_norm, ReLUWS))
                nc_block_in = nc_out
        else:
            self.blocks = None

    def _parse_conv_nn(self, up_conv_nn, stride, N):
        if _is_list(up_conv_nn[0]):
            up_conv_nn = up_conv_nn[0]
        expected = 2 if self.skip_first else 3
        assert len(up_conv_nn) == expected, \
            f"ResNetUp with skip_first={self.skip_first} expects up_conv_nn to have length of {expected} but got " \
            f"len(up_conv_nn)={len(up_conv_nn)}."
        if self.skip_first:
            nc_in, nc_out = up_conv_nn
            nc_skip_in = 0
        else:
            nc_in, nc_skip_in, nc_out = up_conv_nn
        nc_stride_out = nc_in if _single(stride, "stride") > 1 and N > 0 else nc_out
        nc_block_in = nc_stride_out if self.skip_first else nc_stride_out + nc_skip_in
        return nc_in, nc_stride_out, nc_block_in, nc_out

    def output_hw(self, H, W):
        """Spatial size of the output for an H x W input."""
        if self.conv_in is None:
            return H, W
        return ops.convt_out_hw(self._kind, H, W)

    def _skip_hw(self, H, W, skip_hw, where="ResNetUp"):
        """The size the skip connection must have: the input's (skip_first) or the upsampled map's."""
        hw = (H, W) if self.skip_first or self.conv_in is None else self.output_hw(H, W)
        if skip_hw is not None and tuple(skip_hw) != tuple(hw):
            raise ValueError(f"{where}: the skip connection is {skip_hw[0]}x{skip_hw[1]} but the map it joins is "
                             f"{hw[0]}x{hw[1]}; the image sides must be multiples of 2 ** (number of strided "
                             f"stages)")

    def forward_rows(self, x, skip):
        """The stage on channels-last rows: x [B, H, W, C_in], skip [B, H', W', C_skip] or None."""
        self._skip_hw(x.shape[1], x.shape[2], None if skip is None else skip.shape[1:3])
        if self.skip_first and skip is not None:
            x = torch.cat((x.float(), skip.float()), dim=3)
        if self.conv_in is not None:
            conv, norm, _ = self.conv_in
            x = ops.convt_gn_relu_ws(x, conv, norm, self._kind)
        if not self.skip_first and skip is not None:
            x = torch.cat((x.float(), skip.float()), dim=3)
        if self.blocks is not None:
            for blk in self.blocks:
                x = ops.res_block_t(x, blk)
        return x

    def forward(self, x, skip, *args, **kwargs):
        h = _rows(x)
        return self.forward_rows(h, None if skip is None else _rows(skip)).to(_out_dtype(x)).permute(0, 3, 1, 2)

    def extra_repr(self) -> str:
        return f"skip_first={self.skip_first}"


class Dropout2d(nn.Dropout2d):
    """Dropout2d with kwargs support (image.py:479-482): F.dropout2d, one Bernoulli draw per (image, channel)."""

    def forward(self, input, *args, **kwargs):
        return super().forward(input)

    def draw_mask(self, x, reset=True):
        """The [B, C, 1, 1] mask F.dropout2d draws for x [B, C, H, W] (the same torch RNG calls), or None when it is
        the identity."""
        if not self.training or not self.p:
            return None
        return x.new_empty(x.shape[0], x.shape[1], 1, 1).bernoulli_(1 - self.p).div_(1 - self.p)


class PersistentDropout2d(nn.Module):
    """Dropout2d whose [1, C, 1, 1] mask is kept across calls until reset (image.py:485-525); the identity, and no
    mask, in eval mode."""

    def __init__(self, input_nc, p=0.5):
        self.input_nc = input_nc
        self.p = p
        self.mask = None
        super().__init__()

    def draw_mask(self, x, reset=True):
        if not self.training or not self.p:
            self.mask = None
            return None
        if self.mask is None or reset:
            mask = x.new_empty(1, self.input_nc, 1, 1, requires_grad=False)
            mask = mask.bernoulli_(1 - self.p)
            self.mask = mask.div_(1 - self.p)
        return self.mask

    def forward(self, x, reset, *args, **kwargs):
        mask = self.draw_mask(x, reset)
        return x if mask is None else x * mask.expand_as(x)

    def extra_repr(self) -> str:
        return f"input_nc={self.input_nc}, p={self.p}"


class UnaryConv(nn.Module):
    """Dropout -- 1x1 convolution -- activation -- dropout on images (image.py:408-476), the last convolution of
    UNet.  The 1x1 runs on libdva_conv2d.so (weight-standardised or not); the dropout masks multiply the channels-last
    rows.  normalization must be None (the reference's own norm path cannot run: it calls the normalization class
    on the tensor)."""

    def __init__(self, input_nc, output_nc, normalization=None, activation=None, weight_standardization=False,
                 in_drop=0, out_drop=0, persistent_drop=False):
        super().__init__()
        if normalization is not None:
            raise NotImplementedError(f"normalization={normalization!r}: only None is supported")
        if activation not in (None, "ReLU"):
            raise NotImplementedError(f"activation={activation!r}: only None and 'ReLU' are supported")
        if in_drop is None or in_drop <= 0:
            self.input_dropout = None
        elif persistent_drop:
            self.input_dropout = PersistentDropout2d(input_nc, p=in_drop)
        else:
            self.input_dropout = Dropout2d(p=in_drop, inplace=True)
        self.norm = None
        if weight_standardization:
            self.conv = Conv2dWS(input_nc, output_nc, stride=1, kernel_size=1)
            self.activation = ReLUWS if activation is not None else None
        else:
            self.conv = nn.Conv2d(input_nc, output_nc, stride=1, kernel_size=1)
            self.activation = nn.ReLU if activation is not None else None
        self._standardize = bool(weight_standardization)
        if out_drop is None or out_drop <= 0:
            self.output_dropout = None
        elif persistent_drop:
            self.output_dropout = PersistentDropout2d(output_nc, p=out_drop)
        else:
            self.output_dropout = Dropout2d(p=out_drop, inplace=True)

    @staticmethod
    def _drop(h, dropout, reset):
        """h [B, H, W, C] times the mask of `dropout` (drawn for the NCHW view of h), or h."""
        if dropout is None:
            return h
        mask = dropout.draw_mask(h.permute(0, 3, 1, 2), reset)
        return h if mask is None else h * mask.reshape(mask.shape[0], 1, 1, mask.shape[1])

    def forward_rows(self, h, reset=True):
        h = self._drop(h, self.input_dropout, reset)
        scale = 0.0 if self.activation is None else (ReLUWS._SCALE if self.activation is ReLUWS else 1.0)
        h = ops.unary_conv(h, self.conv, self._standardize, scale)
        return self._drop(h, self.output_dropout, reset)

    def forward(self, x, *args, **kwargs):
        reset = kwargs.get("reset", args[0] if args else True)
        return self.forward_rows(_rows(x), bool(reset)).to(_out_dtype(x)).permute(0, 3, 1, 2)


SPECIAL_NAMES = ["block_names"]


def fetch_arguments_from_list(opt, index, special_names):
    """The arguments of layer `index` from a compact config (torch_points3d/utils/config.py:78-103): a list-valued
    key gives its index-th entry under the key without a trailing 's' (except special_names), a string entry is
    eval'ed where it parses (config arithmetic), and any other key is passed as it is."""
    args = {}
    for o, v in opt.items():
        name = str(o)
        if _is_list(v) and len(v) > 0:
            if name[-1] == "s" and name not in special_names:
                name = name[:-1]
            v_index = v[index]
            if _is_list(v_index):
                v_index = list(v_index)
            try:
                v_index = eval(v_index)
            except Exception:
                pass
            args[name] = v_index
        else:
            if _is_list(v):
                v = list(v)
            args[name] = v
    return args


def _opt(opt, key):
    """opt[key] for an omegaconf DictConfig, a dict or an attribute dict; None when absent."""
    if hasattr(opt, "get"):
        return opt.get(key)
    return getattr(opt, key, None)


class UNet(nn.Module):
    """The image UNet of the reference (image.py:531-627): ResNetDown stages, ResNetUp stages joined by symmetric
    skip connections, and an optional UnaryConv, built from the compact config format (down_conv.down_conv_nn,
    up_conv.up_conv_nn, optional last_conv).  Input [B, C, H, W] on CUDA; output [B, C', H', W'] with channels-last
    strides in the input's dtype (fp32 under autocast).  Called as conv(x, reset): reset (default True) draws a new
    persistent dropout mask in last_conv."""

    def __init__(self, opt):
        super().__init__()
        down, up = _opt(opt, "down_conv"), _opt(opt, "up_conv")
        if down is None or up is None or _is_list(down) or "down_conv_nn" not in down or _is_list(up) \
                or "up_conv_nn" not in up:
            raise NotImplementedError("UNet: only the compact format (down_conv.down_conv_nn and up_conv.up_conv_nn) "
                                      "is supported")
        self._init_from_compact_format(opt)

    def _init_from_compact_format(self, opt):
        down, up = _opt(opt, "down_conv"), _opt(opt, "up_conv")
        self.down_modules = nn.ModuleList()
        for i in range(len(down["down_conv_nn"])):
            self.down_modules.append(self._build_module(down, i, "DOWN"))
        if _opt(opt, "innermost") is not None:
            raise NotImplementedError("innermost: the BottleneckBlock inner module is not supported")
        self.inner_modules = None
        self.up_modules = nn.ModuleList()
        for i in range(len(up["up_conv_nn"])):
            self.up_modules.append(self._build_module(up, i, "UP"))
        last = _opt(opt, "last_conv")
        self.last = self._build_module(last, 0, "LAST") if last is not None else None

    def _build_module(self, opt, index, flow):
        module_cls = {"down": ResNetDown, "up": ResNetUp, "last": UnaryConv}.get(flow.lower())
        if module_cls is None:
            raise NotImplementedError(f"flow={flow!r}")
        return module_cls(**fetch_arguments_from_list(opt, index, SPECIAL_NAMES))

    def check_sizes(self, H, W):
        """The spatial size of the output for an H x W input; ValueError, naming the stage and both shapes, where a
        skip connection would not match the map it joins (the sides are not multiples of 2 ** strided stages)."""
        sizes = []
        for m in self.down_modules:
            H, W = m.output_hw(H, W)
            sizes.append((H, W))
        stack = sizes[:-1]
        if self.up_modules[0].skip_first:
            stack.append(None)
        for i, m in enumerate(self.up_modules):
            skip = stack.pop(-1) if stack else None
            m._skip_hw(H, W, skip, where=f"UNet up stage {i}")
            H, W = m.output_hw(H, W)
        return H, W

    def forward(self, x, *args, **kwargs):
        reset = kwargs.get("reset", args[0] if args else True)
        self.check_sizes(x.shape[2], x.shape[3])
        h = x.float() if x.is_floating_point() else x
        stack = []
        for m in self.down_modules[:-1]:
            h = m(h)
            stack.append(h)
        h = self.down_modules[-1](h)
        if self.up_modules[0].skip_first:
            stack.append(None)
        h = _rows(h)
        for m in self.up_modules:
            skip = stack.pop(-1) if stack else None
            h = m.forward_rows(h, None if skip is None else _rows(skip))
        if self.last is not None:
            h = self.last.forward_rows(h, bool(reset))
        return h.to(_out_dtype(x)).permute(0, 3, 1, 2)


# --------------------------------------------------------------------------------------------------------------------
# ResNet-18 pretrained on ADE20K (mit_semseg's resnet18dilated) behind the reference's wrappers (image.py:793-956), on
# the sm_90a kernels of libdva_resnet.so.  The module tree, parameter and buffer names are the reference's, so a
# reference DeepViewAgg checkpoint loads with strict=True; the convolutions and BatchNorms only hold the parameters.
# --------------------------------------------------------------------------------------------------------------------
class SynchronizedBatchNorm2d(nn.BatchNorm2d):
    """Parameters and buffers of mit_semseg's SynchronizedBatchNorm2d.  On one device its forward is
    F.batch_norm(x, running_mean, running_var, weight, bias, training, momentum, eps): num_batches_tracked never moves
    and the momentum is 0.001.  The three extra buffers are in the state dict and never touched on one device."""

    steps_counter = False   # ops._bn_cfg: num_batches_tracked stays where it is

    def __init__(self, num_features, eps=1e-5, momentum=0.001, affine=True):
        super().__init__(num_features, eps=eps, momentum=momentum, affine=affine)
        self.register_buffer('_tmp_running_mean', torch.zeros(num_features))
        self.register_buffer('_tmp_running_var', torch.ones(num_features))
        self.register_buffer('_running_iter', torch.ones(1))

    def forward(self, input):
        raise NotImplementedError("SynchronizedBatchNorm2d runs fused with its convolution: call the "
                                  "ADE20KResNet18* module that holds it")


class FusedBatchNorm2d(nn.BatchNorm2d):
    """Parameters and buffers of a plain nn.BatchNorm2d of the ImageNet and Cityscapes trunks (momentum 0.1 or None,
    num_batches_tracked += 1 per training forward, as torch's); it runs fused with its convolution."""

    def forward(self, input):
        raise NotImplementedError("FusedBatchNorm2d runs fused with its convolution: call the ResNet18* or "
                                  "CityscapesResNet18* module that holds it")


class FusedConv2d(nn.Conv2d):
    """Parameters of a bias-free convolution of the ResNet-18 trunk; it runs fused with its BatchNorm and ReLU."""

    def forward(self, input):
        raise NotImplementedError("FusedConv2d runs fused with its BatchNorm: call the ADE20KResNet18* module that "
                                  "holds it")


class FusedReLU(nn.ReLU):
    """ReLU of the ResNet-18 trunk; fused into the BatchNorm pass."""

    def forward(self, input):
        raise NotImplementedError("FusedReLU runs fused with its BatchNorm: call the ADE20KResNet18* module that "
                                  "holds it")


class FusedMaxPool2d(nn.MaxPool2d):
    """MaxPool2d(3, stride 2, padding 1 or 0) of a stem; run by the ResNet-18 module that holds it."""

    def __init__(self, padding=1):
        super().__init__(kernel_size=3, stride=2, padding=padding)

    def forward(self, input):
        raise NotImplementedError("FusedMaxPool2d is run by the ResNet-18 module that holds it")


def _conv3x3(c_in, c_out, stride=1, dilation=1):
    return FusedConv2d(c_in, c_out, kernel_size=3, stride=stride, padding=dilation, dilation=dilation, bias=False)


class BasicBlock(nn.Module):
    """mit_semseg's, torchvision's and the Cityscapes BasicBlock: relu(bn2(conv2(relu(bn1(conv1 x)))) + residual),
    the residual x or downsample = (1x1 conv, BN); `norm` is the BatchNorm class.  Runs as one node
    (ops.rn_basic_block)."""

    def __init__(self, inplanes, planes, stride=1, dilation=(1, 1), downsample=None, norm=SynchronizedBatchNorm2d):
        super().__init__()
        self.conv1 = _conv3x3(inplanes, planes, stride, dilation[0])
        self.bn1 = norm(planes)
        self.relu = FusedReLU(inplace=True)
        self.conv2 = _conv3x3(planes, planes, 1, dilation[1])
        self.bn2 = norm(planes)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        return ops.rn_basic_block(x, self)


def _make_layer(inplanes, planes, stride, dilations=(1, 1), norm=SynchronizedBatchNorm2d):
    """Two BasicBlocks as resnet18dilated has them after _nostride_dilate: dilations of (block 0 conv1, every other
    3x3); the downsample 1x1 has the block's stride."""
    ds = None
    if stride != 1 or inplanes != planes:
        ds = nn.Sequential(FusedConv2d(inplanes, planes, kernel_size=1, stride=stride, bias=False), norm(planes))
    d0, d = dilations
    return nn.Sequential(BasicBlock(inplanes, planes, stride, (d0, d), ds, norm),
                         BasicBlock(planes, planes, 1, (d, d), norm=norm))


def _make_trunk_layer(name):
    if name == 'layer0':
        return nn.Sequential(_conv3x3(3, 64, stride=2), SynchronizedBatchNorm2d(64), FusedReLU(inplace=True),
                             _conv3x3(64, 64), SynchronizedBatchNorm2d(64), FusedReLU(inplace=True),
                             _conv3x3(64, 128), SynchronizedBatchNorm2d(128), FusedReLU(inplace=True),
                             FusedMaxPool2d())
    return {'layer1': lambda: _make_layer(128, 64, 1, (1, 1)), 'layer2': lambda: _make_layer(64, 128, 2, (1, 1)),
            'layer3': lambda: _make_layer(128, 256, 1, (1, 2)), 'layer4': lambda: _make_layer(256, 512, 1, (2, 4))}[name]()


def _mit_semseg_init(module):
    """mit_semseg's initialisation: conv weights normal with std sqrt(2 / (k^2 C_out)), BN weight 1 and bias 0."""
    for m in module.modules():
        if isinstance(m, nn.Conv2d):
            n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
            m.weight.data.normal_(0, sqrt(2. / n))
        elif isinstance(m, nn.BatchNorm2d):
            m.weight.data.fill_(1.)
            m.bias.data.zero_()


# positions of mit_semseg's stem modules in layer0
_STEM_KEYS = {'conv1': '0', 'bn1': '1', 'conv2': '3', 'bn2': '4', 'conv3': '6', 'bn3': '7'}
_TRUNK_LAYERS = ['layer0', 'layer1', 'layer2', 'layer3', 'layer4']


def _mit_semseg_keys():
    """Every key of mit_semseg's encoder_epoch_20.pth -> (layer, key inside that layer of the wrapper)."""
    keys = {}
    inverse = {v: k for k, v in _STEM_KEYS.items()}
    for name in _TRUNK_LAYERS:
        for k in _make_trunk_layer(name).state_dict():
            if name == 'layer0':
                head, rest = k.split('.', 1)
                keys[f"{inverse[head]}.{rest}"] = (name, k)
            else:
                keys[f"{name}.{k}"] = (name, k)
    return keys


def load_mit_semseg_encoder(module, state_dict):
    """Load mit_semseg's resnet18dilated encoder state dict (encoder_epoch_20.pth: conv1, bn1, ..., layer4.1.bn2.*)
    into the layers an ADE20KResNet18* module holds (its conv.<i>.*).  The state dict must have exactly the
    checkpoint's keys; a missing or extra key raises KeyError.
    Load before nn.SyncBatchNorm.convert_sync_batchnorm: the loader expects the unconverted BatchNorm classes."""
    mapping = _mit_semseg_keys()
    missing = sorted(set(mapping) - set(state_dict))
    extra = sorted(set(state_dict) - set(mapping))
    if missing or extra:
        raise KeyError(f"not a mit_semseg resnet18dilated encoder state dict: missing {missing[:5]}"
                       f"{' ...' if len(missing) > 5 else ''}, unexpected {extra[:5]}{' ...' if len(extra) > 5 else ''}")
    position = {name: i for i, name in enumerate(module._LAYERS)}
    ours = {f"conv.{position[layer]}.{k}": state_dict[key] for key, (layer, k) in mapping.items() if layer in position}
    module.load_state_dict(ours, strict=True)
    return module


def _check_bn_values(bn, training, B, H, W):
    """torch's error for a training BatchNorm that would see one value per channel, raised before any launch.  A
    BatchNorm synchronised over ranks (ops.bn_sync_group) counts the values of every rank: ops raises it after its
    all-reduce, on every rank at once."""
    if ops.bn_sync_group(bn) is not None:
        return
    if training and B * H * W <= 1:
        raise ValueError(f"Expected more than 1 value per channel when training, got input size "
                         f"{[B, bn.num_features, H, W]}")


# The BatchNorms a trunk or a pyramid head holds: SynchronizedBatchNorm2d, PrudentSynchronizedBatchNorm2d and
# FusedBatchNorm2d, or the nn.SyncBatchNorm that nn.SyncBatchNorm.convert_sync_batchnorm makes of any of them.
_BATCHNORMS = (nn.BatchNorm2d, nn.SyncBatchNorm)


# A trunk as _run_trunk walks it: a list of layers, each the stem -- a list of (conv, BatchNorm) units, then the
# max pool, of padding `pool_padding` (1 when the list does not say) -- or a Sequential of BasicBlocks.
class _Stem(list):
    """A stem's (conv, BatchNorm) units in order, and the padding of the max pool after them."""

    def __init__(self, units, pool_padding):
        super().__init__(units)
        self.pool_padding = pool_padding


def _stem_of(layer):
    """The stem Sequential of a wrapper (nested Sequentials flattened: convs, BatchNorms, ReLUs, then the max pool) as
    _run_trunk walks it."""
    mods = [m for m in layer.modules() if not isinstance(m, nn.Sequential)]
    convs = [m for m in mods if isinstance(m, nn.Conv2d)]
    bns = [m for m in mods if isinstance(m, _BATCHNORMS)]
    return _Stem(list(zip(convs, bns)), mods[-1].padding)


def _pool_padding(stem):
    return getattr(stem, 'pool_padding', 1)


def _trunk_bn_sizes(trunk, H, W):
    """Yields (BatchNorm, H, W of the map it normalises) along the trunk for an H x W input; ValueError when a max
    pool would get a map smaller than its window."""
    for layer in trunk:
        if isinstance(layer, list):
            for conv, bn in layer:
                H, W = ops.rn_out(H, conv.stride[0]), ops.rn_out(W, conv.stride[0])
                yield bn, H, W
            H, W = ops.rn_pool_out(H, _pool_padding(layer)), ops.rn_pool_out(W, _pool_padding(layer))
        else:
            for block in layer:
                H, W = ops.rn_out(H, block.conv1.stride[0]), ops.rn_out(W, block.conv1.stride[0])
                yield block.bn1, H, W
                yield block.bn2, H, W
                if block.downsample is not None:
                    yield block.downsample[1], H, W


def _run_trunk(trunk, h):
    """Yields the channels-last output of each layer of the trunk for channels-last rows h."""
    for layer in trunk:
        if isinstance(layer, list):
            for conv, bn in layer:
                h = ops.rn_conv_bn_relu(h, conv, bn)
            h = ops.rn_maxpool(h, _pool_padding(layer))
        else:
            for block in layer:
                h = ops.rn_basic_block(h, block)
        yield h


def _load_weights(weights):
    """A state dict, or the file at `weights` loaded on the CPU."""
    return weights if isinstance(weights, dict) else torch.load(weights, map_location='cpu')


class _ResNet18Wrapper(nn.Module):
    """What the reference's ResNet-18 wrappers share (ADE20KResNet18*, ResNet18*, CityscapesResNet18*): `frozen` and
    train(), scale_factor (< 0: conv_scale_factor), input_nc / output_nc / conv_scale_factor, the input checks and
    the trunk walk over self.conv.  A subclass builds self.conv (its _LAYERS) and calls _setup."""
    _LAYERS = _TRUNK_LAYERS

    def _setup(self, frozen, scale_factor):
        # If the model is frozen, it will always remain in eval mode and the parameters will have requires_grad=False
        self.frozen = frozen
        if self.frozen:
            self.training = False

        # scale_factor < 0: resize by conv_scale_factor
        if scale_factor is not None and scale_factor < 0:
            scale_factor = self.conv_scale_factor
        self.scale_factor = scale_factor

    def _check_input(self, x):
        require_cuda(x)
        if x.dim() != 4 or x.shape[1] != self.input_nc:
            raise ValueError(f"{type(self).__name__} expects [B, {self.input_nc}, H, W] images, got shape "
                             f"{tuple(x.shape)}")
        B, _, H, W = x.shape
        for bn, H, W in self._bn_sizes(H, W):
            _check_bn_values(bn, bn.training, B, H, W)

    def _trunk_modules(self):
        return self.conv

    def _trunk(self):
        return [layer if isinstance(layer[0], BasicBlock) else _stem_of(layer) for layer in self._trunk_modules()]

    def _bn_sizes(self, H, W):
        """Yields (BatchNorm, H, W of the map it normalises) along the trunk for an H x W input."""
        return _trunk_bn_sizes(self._trunk(), H, W)

    def _layers(self, h):
        """Yields the channels-last output of each layer of the trunk for channels-last rows h."""
        return _run_trunk(self._trunk(), h)

    def forward(self, x, *args, **kwargs):
        self._check_input(x)
        for h in self._layers(_rows(x)):
            pass
        if self.scale_factor is not None:
            size = (int(h.shape[1] * float(self.scale_factor)), int(h.shape[2] * float(self.scale_factor)))
            h = ops.rn_resize([h], size, scale_factor=float(self.scale_factor))
        return h.to(_out_dtype(x)).permute(0, 3, 1, 2)

    @property
    def input_nc(self):
        return self._LAYERS_IN[self._LAYERS[0]]

    @property
    def output_nc(self):
        return self._LAYERS_OUT[self._LAYERS[-1]]

    @property
    def conv_scale_factor(self):
        return torch.prod(torch.LongTensor([self._LAYERS_SCALE[s] for s in self._LAYERS])).item()

    @property
    def frozen(self):
        return self._frozen

    @frozen.setter
    def frozen(self, frozen):
        if isinstance(frozen, bool):
            self._frozen = frozen
        for p in self.parameters():
            p.requires_grad = not self.frozen

    def train(self, mode=True):
        return super().train(mode and not self.frozen)

    def extra_repr(self) -> str:
        return f"scale_factor={self.scale_factor}" if self.scale_factor is not None else ""


class _Pyramid:
    """The Pyramid forward of the wrappers: every layer's output resized to int(side * scale_factor /
    conv_scale_factor) of the input sides (a size-based bilinear resize) and concatenated along the channels,
    written into one buffer."""

    def __init__(self, frozen=False, scale_factor=-1, **kwargs):
        assert scale_factor is not None, f'scale_factor cannot be None for feature pyramid.'
        super().__init__(frozen=frozen, scale_factor=scale_factor, **kwargs)

    def forward(self, x, *args, **kwargs):
        self._check_input(x)
        size = [int(s * self.scale_factor / self.conv_scale_factor) for s in x.shape[2:4]]
        h = ops.rn_resize(list(self._layers(_rows(x))), size)
        return h.to(_out_dtype(x)).permute(0, 3, 1, 2)


class ADE20KResNet18TruncatedLayer4(_ResNet18Wrapper):
    """ResNet-18 encoder pretrained on ADE20K (mit_semseg's resnet18dilated), truncated after `_LAYERS`
    (image.py:793-898), on the sm_90a kernels of libdva_resnet.so.

    weights: None (mit_semseg's random initialisation), a path to mit_semseg's encoder_epoch_20.pth or its state
    dict (load_mit_semseg_encoder).  The reference always loads that checkpoint from its own tree.
    Input [B, 3, H, W] on CUDA (input_nc channels), NCHW or channels-last; output [B, output_nc, H', W'] in the
    input's dtype (fp32 under autocast) with channels-last strides.  Each BatchNorm runs in its own mode (its
    .training): batch statistics and a running-stat update (momentum 0.001) in training mode, the running stats in
    eval mode."""
    _LAYERS = ['layer0', 'layer1', 'layer2', 'layer3', 'layer4']
    _LAYERS_IN = {k: v for k, v in zip(_TRUNK_LAYERS, [3, 128, 64, 128, 256])}
    _LAYERS_OUT = {k: v for k, v in zip(_TRUNK_LAYERS, [128, 64, 128, 256, 512])}
    _LAYERS_SCALE = {k: v for k, v in zip(_TRUNK_LAYERS, [4, 1, 2, 1, 1])}

    def __init__(self, frozen=False, scale_factor=None, weights=None, **kwargs):
        super().__init__()
        self.conv = nn.Sequential(*[_make_trunk_layer(layer) for layer in self._LAYERS])
        _mit_semseg_init(self.conv)
        if weights is not None:
            load_mit_semseg_encoder(self, _load_weights(weights))
        self._setup(frozen, scale_factor)


class ADE20KResNet18TruncatedLayer0(ADE20KResNet18TruncatedLayer4):
    _LAYERS = ['layer0']


class ADE20KResNet18TruncatedLayer1(ADE20KResNet18TruncatedLayer4):
    _LAYERS = ['layer0', 'layer1']


class ADE20KResNet18TruncatedLayer2(ADE20KResNet18TruncatedLayer4):
    _LAYERS = ['layer0', 'layer1', 'layer2']


class ADE20KResNet18TruncatedLayer3(ADE20KResNet18TruncatedLayer4):
    _LAYERS = ['layer0', 'layer1', 'layer2', 'layer3']


class ADE20KResNet18Layer0(ADE20KResNet18TruncatedLayer4):
    _LAYERS = ['layer0']


class ADE20KResNet18Layer1(ADE20KResNet18TruncatedLayer4):
    _LAYERS = ['layer1']


class ADE20KResNet18Layer2(ADE20KResNet18TruncatedLayer4):
    _LAYERS = ['layer2']


class ADE20KResNet18Layer3(ADE20KResNet18TruncatedLayer4):
    _LAYERS = ['layer3']


class ADE20KResNet18Layer4(ADE20KResNet18TruncatedLayer4):
    _LAYERS = ['layer4']


class ADE20KResNet18Pyramid(_Pyramid, ADE20KResNet18TruncatedLayer4):
    """Every layer's output resized to int(side * scale_factor / conv_scale_factor) of the input sides and
    concatenated: 128 + 64 + 128 + 256 + 512 = 1088 channels, written into one buffer."""


# --------------------------------------------------------------------------------------------------------------------
# torchvision's ImageNet ResNet-18 (ResNet18*, image.py:959-1126) and the Cityscapes ResNet-18 of SFSegNets
# (CityscapesResNet18*, image.py:1129-1399) on the same kernels and trunk walk.  Both use plain nn.BatchNorm2d
# (momentum 0.1, num_batches_tracked += 1 per training forward) and no dilation.  ImageNet layer0 is (7x7/2 conv, BN,
# ReLU, MaxPool2d(3, 2, 1)); Cityscapes layer0 is (Sequential(3x3/2 conv, BN, ReLU, 3x3 conv, BN, ReLU, 3x3 conv),
# BN, ReLU, MaxPool2d(3, 2, 0)), whose last row and column can belong to no window.
# --------------------------------------------------------------------------------------------------------------------
def _make_imagenet_layer(name):
    if name == 'layer0':
        return nn.Sequential(FusedConv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False), FusedBatchNorm2d(64),
                             FusedReLU(inplace=True), FusedMaxPool2d(padding=1))
    inplanes, planes, stride = {'layer1': (64, 64, 1), 'layer2': (64, 128, 2), 'layer3': (128, 256, 2),
                                'layer4': (256, 512, 2)}[name]
    return _make_layer(inplanes, planes, stride, norm=FusedBatchNorm2d)


def _make_cityscapes_layer(name):
    if name == 'layer0':
        stem = nn.Sequential(_conv3x3(3, 64, stride=2), FusedBatchNorm2d(64), FusedReLU(inplace=True),
                             _conv3x3(64, 64), FusedBatchNorm2d(64), FusedReLU(inplace=True), _conv3x3(64, 128))
        return nn.Sequential(stem, FusedBatchNorm2d(128), FusedReLU(inplace=True), FusedMaxPool2d(padding=0))
    inplanes, planes, stride = {'layer1': (128, 64, 1), 'layer2': (64, 128, 2), 'layer3': (128, 256, 2),
                                'layer4': (256, 512, 2)}[name]
    return _make_layer(inplanes, planes, stride, norm=FusedBatchNorm2d)


def _kaiming_init(module):
    """torchvision's and SFSegNets' initialisation: conv weights kaiming_normal_ (fan_out, relu), BN weight 1 and
    bias 0."""
    for m in module.modules():
        if isinstance(m, nn.Conv2d):
            nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
        elif isinstance(m, nn.BatchNorm2d):
            nn.init.constant_(m.weight, 1)
            nn.init.constant_(m.bias, 0)


def _check_keys(what, expected, state_dict, optional=()):
    """KeyError unless state_dict has every key of `expected` and nothing outside expected | optional."""
    missing = sorted(set(expected) - set(state_dict))
    extra = sorted(set(state_dict) - set(expected) - set(optional))
    if missing or extra:
        raise KeyError(f"not a {what} state dict: missing {missing[:5]}{' ...' if len(missing) > 5 else ''}, "
                       f"unexpected {extra[:5]}{' ...' if len(extra) > 5 else ''}")


def _load_layers(module, state_dict):
    """Load {layer name: {key inside the layer: tensor}} into the layers `module` holds (conv.<i>.* of a wrapper,
    layer<i>.* of CityscapesResNet18) with strict=True."""
    position = {name: i for i, name in enumerate(module._LAYERS)}
    prefix = (lambda name: f"conv.{position[name]}.") if hasattr(module, 'conv') else (lambda name: f"{name}.")
    module.load_state_dict({prefix(layer) + k: v for (layer, k), v in state_dict.items() if layer in position},
                           strict=True)
    return module


def _torchvision_resnet18_keys():
    """Every key of torchvision's resnet18 state dict -> (layer, key inside that layer of the wrapper); fc -> None."""
    keys = {'fc.weight': None, 'fc.bias': None}
    for name in _TRUNK_LAYERS:
        for k in _make_imagenet_layer(name).state_dict():
            if name == 'layer0':
                head, rest = k.split('.', 1)
                keys[f"{ {'0': 'conv1', '1': 'bn1'}[head]}.{rest}"] = (name, k)
            else:
                keys[f"{name}.{k}"] = (name, k)
    return keys


def load_torchvision_resnet18(module, state_dict):
    """Load torchvision's ImageNet resnet18 state dict (conv1, bn1, layer1..layer4, fc) into the layers a ResNet18*
    module holds; fc is dropped.  The state dict must have exactly torchvision's keys, except that
    num_batches_tracked may be missing, as in checkpoints saved before torch 0.4.1: those counters are left as they
    are, as torch's BatchNorm loads such a checkpoint.  A missing or extra key raises KeyError.
    Load before nn.SyncBatchNorm.convert_sync_batchnorm: the loader expects the unconverted BatchNorm classes."""
    mapping = _torchvision_resnet18_keys()
    counters = [k for k in mapping if k.endswith('.num_batches_tracked')]
    _check_keys("torchvision resnet18", [k for k in mapping if k not in counters], state_dict, counters)
    own = module.state_dict()
    position = {name: i for i, name in enumerate(module._LAYERS)}
    return _load_layers(module, {target: state_dict[key] if key in state_dict else
                                 own[f"conv.{position[target[0]]}.{target[1]}"]
                                 for key, target in mapping.items() if target is not None and target[0] in position})


def _cityscapes_resnet18_keys():
    """Every key of SFSegNets' resnet18_SFSegNets.pth (CityscapesResNet18's state dict) -> (layer, key inside it)."""
    return {f"{name}.{k}": (name, k) for name in _TRUNK_LAYERS for k in _make_cityscapes_layer(name).state_dict()}


def load_cityscapes_resnet18(module, state_dict):
    """Load SFSegNets' Cityscapes ResNet-18 state dict (resnet18_SFSegNets.pth: layer0.0.0.weight, ...,
    layer4.1.bn2.*, 138 keys) into CityscapesResNet18 or the layers a CityscapesResNet18* module holds.  The state
    dict must have exactly those keys; a missing or extra key raises KeyError.
    Load before nn.SyncBatchNorm.convert_sync_batchnorm: the loader expects the unconverted BatchNorm classes."""
    mapping = _cityscapes_resnet18_keys()
    _check_keys("Cityscapes ResNet-18 (resnet18_SFSegNets.pth)", mapping, state_dict)
    return _load_layers(module, {target: state_dict[key] for key, target in mapping.items()})


class ResNet18TruncatedLayer4(_ResNet18Wrapper):
    """torchvision's ImageNet ResNet-18, truncated after `_LAYERS` (image.py:992-1066), on the sm_90a kernels of
    libdva_resnet.so; layer0 is (conv1 7x7/2, bn1, relu, maxpool 3/2/1).

    weights: None (torchvision's random initialisation), a path to torchvision's resnet18 state dict or the dict
    (load_torchvision_resnet18).  `pretrained`, like any other unused config key, is swallowed: the reference loads
    the checkpoint from its own tree.  Input [B, 3, H, W] on CUDA (input_nc channels), NCHW or channels-last; output
    [B, output_nc, H', W'] in the input's dtype (fp32 under autocast) with channels-last strides.  Each BatchNorm
    runs in its own mode: batch statistics, a running-stat update with its momentum (None: the cumulative average)
    and num_batches_tracked += 1 in training mode, the running stats in eval mode."""
    _LAYERS_IN = {k: v for k, v in zip(_TRUNK_LAYERS, [3, 64, 64, 128, 256])}
    _LAYERS_OUT = {k: v for k, v in zip(_TRUNK_LAYERS, [64, 64, 128, 256, 512])}
    _LAYERS_SCALE = {k: v for k, v in zip(_TRUNK_LAYERS, [4, 1, 2, 2, 2])}
    _make = staticmethod(_make_imagenet_layer)
    _load = staticmethod(load_torchvision_resnet18)

    def __init__(self, frozen=False, scale_factor=None, weights=None, **kwargs):
        super().__init__()
        self.conv = nn.Sequential(*[self._make(layer) for layer in self._LAYERS])
        _kaiming_init(self.conv)
        if weights is not None:
            self._load(self, _load_weights(weights))
        self._setup(frozen, scale_factor)


class ResNet18TruncatedLayer0(ResNet18TruncatedLayer4):
    _LAYERS = ['layer0']


class ResNet18TruncatedLayer1(ResNet18TruncatedLayer4):
    _LAYERS = ['layer0', 'layer1']


class ResNet18TruncatedLayer2(ResNet18TruncatedLayer4):
    _LAYERS = ['layer0', 'layer1', 'layer2']


class ResNet18TruncatedLayer3(ResNet18TruncatedLayer4):
    _LAYERS = ['layer0', 'layer1', 'layer2', 'layer3']


class ResNet18Layer0(ResNet18TruncatedLayer4):
    _LAYERS = ['layer0']


class ResNet18Layer1(ResNet18TruncatedLayer4):
    _LAYERS = ['layer1']


class ResNet18Layer2(ResNet18TruncatedLayer4):
    _LAYERS = ['layer2']


class ResNet18Layer3(ResNet18TruncatedLayer4):
    _LAYERS = ['layer3']


class ResNet18Layer4(ResNet18TruncatedLayer4):
    _LAYERS = ['layer4']


class ResNet18Pyramid(_Pyramid, ResNet18TruncatedLayer4):
    """Every layer's output resized to the input size (scale_factor -1) and concatenated: 64 + 64 + 128 + 256 + 512 =
    1024 channels, written into one buffer."""


class CityscapesResNet18TruncatedLayer4(ResNet18TruncatedLayer4):
    """The Cityscapes ResNet-18 of SFSegNets, truncated after `_LAYERS` (image.py:1268-1339); layer0 is
    (Sequential(conv 3x3/2, bn, relu, conv, bn, relu, conv), bn, relu, maxpool 3/2/0).  The maxpool keeps
    floor((side - 3) / 2) + 1 of each side, so an image whose stem output is smaller than 3 raises ValueError.

    weights: None (SFSegNets' random initialisation), a path to resnet18_SFSegNets.pth or its state dict
    (load_cityscapes_resnet18).  Otherwise as ResNet18TruncatedLayer4."""
    _LAYERS_IN = {k: v for k, v in zip(_TRUNK_LAYERS, [3, 128, 64, 128, 256])}
    _LAYERS_OUT = {k: v for k, v in zip(_TRUNK_LAYERS, [128, 64, 128, 256, 512])}
    _make = staticmethod(_make_cityscapes_layer)
    _load = staticmethod(load_cityscapes_resnet18)


class CityscapesResNet18TruncatedLayer0(CityscapesResNet18TruncatedLayer4):
    _LAYERS = ['layer0']


class CityscapesResNet18TruncatedLayer1(CityscapesResNet18TruncatedLayer4):
    _LAYERS = ['layer0', 'layer1']


class CityscapesResNet18TruncatedLayer2(CityscapesResNet18TruncatedLayer4):
    _LAYERS = ['layer0', 'layer1', 'layer2']


class CityscapesResNet18TruncatedLayer3(CityscapesResNet18TruncatedLayer4):
    _LAYERS = ['layer0', 'layer1', 'layer2', 'layer3']


class CityscapesResNet18Layer0(CityscapesResNet18TruncatedLayer4):
    _LAYERS = ['layer0']


class CityscapesResNet18Layer1(CityscapesResNet18TruncatedLayer4):
    _LAYERS = ['layer1']


class CityscapesResNet18Layer2(CityscapesResNet18TruncatedLayer4):
    _LAYERS = ['layer2']


class CityscapesResNet18Layer3(CityscapesResNet18TruncatedLayer4):
    _LAYERS = ['layer3']


class CityscapesResNet18Layer4(CityscapesResNet18TruncatedLayer4):
    _LAYERS = ['layer4']


class CityscapesResNet18Pyramid(_Pyramid, CityscapesResNet18TruncatedLayer4):
    """Every layer's output resized to the input size (scale_factor -1) and concatenated: 128 + 64 + 128 + 256 + 512
    = 1088 channels, written into one buffer."""


class CityscapesResNet18(CityscapesResNet18TruncatedLayer4):
    """The whole Cityscapes ResNet-18 under SFSegNets' names (image.py:1175-1265): layer0..layer4 attributes, so
    resnet18_SFSegNets.pth loads into it as it is; forward returns layer4's output (/32), without resize."""

    def __init__(self, *args, frozen=False, weights=None, **kwargs):
        nn.Module.__init__(self)
        for name in _TRUNK_LAYERS:
            setattr(self, name, _make_cityscapes_layer(name))
        _kaiming_init(self)
        if weights is not None:
            load_cityscapes_resnet18(self, _load_weights(weights))
        self._setup(frozen, None)

    def _trunk_modules(self):
        return [getattr(self, name) for name in _TRUNK_LAYERS]

    def extra_repr(self) -> str:
        return ""


# --------------------------------------------------------------------------------------------------------------------
# ResNet-18 + pyramid pooling pretrained on ADE20K (mit_semseg's resnet18dilated-ppm_deepsup) behind the reference's
# ADE20KResNet18PPM (image.py:634-790): the trunk above under mit_semseg's flat names, and PPMFeatMap, the PPMDeepsup
# decoder without its classifiers, run as one node (ops.rn_ppm_head).
# --------------------------------------------------------------------------------------------------------------------
class FusedAdaptiveAvgPool2d(nn.AdaptiveAvgPool2d):
    """AdaptiveAvgPool2d of a pyramid branch; run by the PPMFeatMap that holds it."""

    def forward(self, input):
        raise NotImplementedError("FusedAdaptiveAvgPool2d is run by the PPMFeatMap that holds it")


class PrudentSynchronizedBatchNorm2d(SynchronizedBatchNorm2d):
    """SynchronizedBatchNorm2d that runs in eval mode for a (1, C, 1, 1) input (image.py:634-656): in a pyramid
    branch, the scale-1 branch at batch size 1 normalises with the running stats and leaves them unchanged."""

    def forward(self, input):
        raise NotImplementedError("PrudentSynchronizedBatchNorm2d runs fused with its convolution: call the "
                                  "PPMFeatMap that holds it")


class ResnetDilated(nn.Module):
    """mit_semseg's ResnetDilated(resnet18, dilate_scale=8) under its flat names (conv1, bn1, relu1, ..., maxpool,
    layer1..layer4), so that encoder_epoch_20.pth loads into it as it is."""

    def __init__(self):
        super().__init__()
        stem = _make_trunk_layer('layer0')
        for name, i in (('conv1', 0), ('bn1', 1), ('relu1', 2), ('conv2', 3), ('bn2', 4), ('relu2', 5),
                        ('conv3', 6), ('bn3', 7), ('relu3', 8), ('maxpool', 9)):
            setattr(self, name, stem[i])
        for name in _TRUNK_LAYERS[1:]:
            setattr(self, name, _make_trunk_layer(name))
        _mit_semseg_init(self)

    def _trunk(self):
        return [[(self.conv1, self.bn1), (self.conv2, self.bn2), (self.conv3, self.bn3)], self.layer1, self.layer2,
                self.layer3, self.layer4]

    def forward(self, x, return_feature_maps=False):
        """mit_semseg's forward: [conv5], or the outputs of layer1..layer4 when return_feature_maps; fp32 maps with
        channels-last strides."""
        outs = [h.permute(0, 3, 1, 2) for h in _run_trunk(self._trunk(), _rows(x))][1:]
        return outs if return_feature_maps else [outs[-1]]


class PPMFeatMap(nn.Module):
    """Pyramid Pooling Module for feature extraction (image.py:659-716): mit_semseg's PPMDeepsup without the deep
    supervision and the classifier.  forward(conv_out, out_size=None) runs on conv_out[-1] ([B, fc_dim, h, w] CUDA)
    as one node (ops.rn_ppm_head) and returns [B, 512, h, w] fp32 with channels-last strides, resized to out_size
    when given."""

    def __init__(self, fc_dim=4096, pool_scales=(1, 2, 3, 6)):
        super().__init__()
        self.ppm = nn.ModuleList([nn.Sequential(FusedAdaptiveAvgPool2d(scale),
                                                FusedConv2d(fc_dim, 512, kernel_size=1, bias=False),
                                                PrudentSynchronizedBatchNorm2d(512), FusedReLU(inplace=True))
                                  for scale in pool_scales])
        self.conv_last = nn.Sequential(FusedConv2d(fc_dim + len(pool_scales) * 512, 512, kernel_size=3, padding=1,
                                                   bias=False),
                                       SynchronizedBatchNorm2d(512), FusedReLU(inplace=True))

    def _check(self, B, h, w, out_size):
        """ValueError, before any launch, where the reference's torch would raise; returns out_size as two ints."""
        for m in self.ppm:
            s = m[0].output_size
            _check_bn_values(m[2], ops.ppm_branch_training(m[2], B, s), B, s, s)
        _check_bn_values(self.conv_last[1], self.conv_last[1].training, B, h, w)
        if out_size is None:
            return None
        if (not isinstance(out_size, (tuple, list, torch.Size)) or len(out_size) != 2
                or not all(isinstance(v, int) and not isinstance(v, bool) and v > 0 for v in out_size)):
            raise ValueError(f"out_size must be two positive ints, got {out_size!r}")
        return tuple(out_size)

    def forward(self, conv_out, *args, out_size=None, **kwargs):
        conv5 = conv_out[-1]
        require_cuda(conv5)
        if conv5.dim() != 4 or conv5.shape[1] != self.ppm[0][1].in_channels:
            raise ValueError(f"PPMFeatMap expects [B, {self.ppm[0][1].in_channels}, h, w] maps, got shape "
                             f"{tuple(conv5.shape)}")
        B, _, h, w = conv5.shape
        out_size = self._check(B, h, w, out_size)
        return ops.rn_ppm_head(_rows(conv5), self, out_size).permute(0, 3, 1, 2)


def _mit_semseg_decoder_init(module):
    """mit_semseg's ModelBuilder.weights_init: conv weights kaiming_normal_, BN weight 1 and bias 1e-4."""
    for m in module.modules():
        if isinstance(m, nn.Conv2d):
            nn.init.kaiming_normal_(m.weight.data)
        elif isinstance(m, nn.BatchNorm2d):
            m.weight.data.fill_(1.)
            m.bias.data.fill_(1e-4)


def _mit_semseg_decoder_keys(fc_dim=512, num_class=150):
    """Every key of mit_semseg's PPMDeepsup decoder_epoch_20.pth -> its shape; PPMFeatMap keeps ppm.* and
    conv_last.0/1.*."""
    keys = {k: tuple(v.shape) for k, v in PPMFeatMap(fc_dim).state_dict().items()}
    keys['cbr_deepsup.0.weight'] = (fc_dim // 4, fc_dim // 2, 3, 3)
    keys.update({f"cbr_deepsup.1.{k}": tuple(v.shape)
                 for k, v in SynchronizedBatchNorm2d(fc_dim // 4).state_dict().items()})
    keys.update({'conv_last.4.weight': (num_class, 512, 1, 1), 'conv_last.4.bias': (num_class,),
                 'conv_last_deepsup.weight': (num_class, fc_dim // 4, 1, 1), 'conv_last_deepsup.bias': (num_class,)})
    return keys


def load_mit_semseg_decoder(module, state_dict):
    """Load mit_semseg's PPMDeepsup decoder state dict (decoder_epoch_20.pth: ppm.*, cbr_deepsup.*, conv_last.*,
    conv_last_deepsup.*) into a PPMFeatMap, or into the decoder of an ADE20KResNet18PPM, keeping what
    PPMFeatMap.from_pretrained keeps: ppm and conv_last[:3].  The state dict must have exactly the checkpoint's keys;
    a missing or extra key raises KeyError.
    Load before nn.SyncBatchNorm.convert_sync_batchnorm: the loader expects the unconverted BatchNorm classes."""
    decoder = getattr(module, 'decoder', module)
    mapping = _mit_semseg_decoder_keys()
    missing = sorted(set(mapping) - set(state_dict))
    extra = sorted(set(state_dict) - set(mapping))
    if missing or extra:
        raise KeyError(f"not a mit_semseg ppm_deepsup decoder state dict: missing {missing[:5]}"
                       f"{' ...' if len(missing) > 5 else ''}, unexpected {extra[:5]}"
                       f"{' ...' if len(extra) > 5 else ''}")
    keep = decoder.state_dict()
    decoder.load_state_dict({k: v for k, v in state_dict.items() if k in keep}, strict=True)
    return module


class ADE20KResNet18PPM(nn.Module):
    """ResNet-18 encoder with the PPM decoder pretrained on ADE20K (mit_semseg's resnet18dilated-ppm_deepsup,
    image.py:719-790), on the sm_90a kernels of libdva_resnet.so and the gather pool of libdva_b200.so.

    weights: None (mit_semseg's random initialisation of both halves) or (encoder, decoder), each a path to or the
    state dict of encoder_epoch_20.pth (loaded into .encoder as it is) and decoder_epoch_20.pth
    (load_mit_semseg_decoder).  `pretrained`, like any other unused config key, is swallowed: the reference always
    loads the checkpoints from its own tree.
    forward(x, out_size=None): x [B, 3, H, W] on CUDA, NCHW or channels-last; output [B, 512, h, w] with h =
    ceil(ceil(ceil(H / 2) / 2) / 2) (the same for w), or [B, 512, *out_size], in the input's dtype (fp32 under
    autocast) with channels-last strides.  Each BatchNorm runs in its own mode, except the Prudent rule of the
    scale-1 branch at batch size 1."""

    def __init__(self, *args, frozen=False, weights=None, **kwargs):
        super().__init__()
        self.encoder = ResnetDilated()
        self.decoder = PPMFeatMap(fc_dim=512)
        _mit_semseg_decoder_init(self.decoder)
        if weights is not None:
            enc, dec = [w if isinstance(w, dict) else torch.load(w, map_location='cpu') for w in weights]
            self.encoder.load_state_dict(enc, strict=True)
            load_mit_semseg_decoder(self, dec)

        # If the model is frozen, it will always remain in eval mode and the parameters will have requires_grad=False
        self.frozen = frozen
        if self.frozen:
            self.training = False

    input_nc = 3
    output_nc = 512

    def forward(self, x, *args, out_size=None, **kwargs):
        require_cuda(x)
        if x.dim() != 4 or x.shape[1] != self.input_nc:
            raise ValueError(f"ADE20KResNet18PPM expects [B, 3, H, W] images, got shape {tuple(x.shape)}")
        B, _, H, W = x.shape
        trunk = self.encoder._trunk()
        for bn, h, w in _trunk_bn_sizes(trunk, H, W):
            _check_bn_values(bn, bn.training, B, h, w)
        out_size = self.decoder._check(B, h, w, out_size)
        for conv5 in _run_trunk(trunk, _rows(x)):
            pass
        y = ops.rn_ppm_head(conv5, self.decoder, out_size)
        return y.to(_out_dtype(x)).permute(0, 3, 1, 2)

    @property
    def frozen(self):
        return self._frozen

    @frozen.setter
    def frozen(self, frozen):
        if isinstance(frozen, bool):
            self._frozen = frozen
        for p in self.parameters():
            p.requires_grad = not self.frozen

    def train(self, mode=True):
        return super().train(mode and not self.frozen)
