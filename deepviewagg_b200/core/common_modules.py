"""MLP building blocks with the reference's parameter names
(torch_points3d/core/common_modules/base_modules.py:38-48, 131-156), so that reference
state_dicts load unchanged: `<mlp>.<i>.0.weight`, `<mlp>.<i>.1.batch_norm.{weight,bias,
running_mean,running_var,num_batches_tracked}`.

The dense projections go through ops.linear (3xTF32 mma.sync kernels for K, N <= 64, wgmma
kernels for wider layers, widths that are not a multiple of 4 zero-padded) -- the only
tensor-core work on this path; BatchNorm uses batch statistics over ALL rows in training.
"""
import torch
from torch import nn


class Identity(nn.Module):
    def forward(self, data):
        return data


class FastBatchNorm1d(nn.Module):
    """BatchNorm over the rows of a [rows, C] (or [B, N, C]) tensor; the wrapped module is
    called `batch_norm` like in the reference (base_modules.py:131-156)."""

    def __init__(self, num_features, momentum=0.1, **kwargs):
        super().__init__()
        self.batch_norm = nn.BatchNorm1d(num_features, momentum=momentum, **kwargs)

    def forward(self, x):
        if x.dim() == 2:
            return self.batch_norm(x)
        if x.dim() == 3:
            return self.batch_norm(x.transpose(1, 2)).transpose(1, 2)
        raise ValueError("Non supported number of dimensions {}".format(x.dim()))


class MLPLayer(nn.Sequential):
    """One `Linear -> FastBatchNorm1d -> activation` layer.  An nn.Sequential (children '0', '1',
    '2': reference parameter names), whose forward fuses BatchNorm + LeakyReLU into two streaming
    passes (ops.batch_norm_act) when the input is a CUDA [rows, C] matrix.  When
    nn.SyncBatchNorm.convert_sync_batchnorm has replaced the inner BatchNorm1d, the projection
    still runs on ops.linear and the nn.SyncBatchNorm module itself normalises, synchronised over
    its process group as torch does it, before the activation."""

    def forward(self, x):
        lin, bn, act = self[0], self[1], self[2]
        if (isinstance(bn, FastBatchNorm1d) and isinstance(bn.batch_norm, nn.SyncBatchNorm)
                and x.dim() == 2 and x.is_cuda and x.shape[0] > 0):
            from .. import ops
            z = ops.linear(x, lin.weight)
            return act(bn(z if lin.bias is None else z + lin.bias))
        fusable = (x.dim() == 2 and x.is_cuda and isinstance(bn, FastBatchNorm1d)
                   and isinstance(act, (nn.LeakyReLU, nn.ReLU, nn.Identity, Identity)) and x.shape[0] > 0)
        if not fusable:
            return super().forward(x)
        slope = act.negative_slope if isinstance(act, nn.LeakyReLU) else (0.0 if isinstance(act, nn.ReLU) else 1.0)
        from .. import ops
        if lin.bias is None:      # every MLP of the pools (bias=False): statistics fused into the GEMM when possible
            return ops.linear_bn_act(x, lin.weight, bn.batch_norm, negative_slope=slope)
        z = ops.linear(x, lin.weight) + lin.bias
        return ops.batch_norm_act(z, bn.batch_norm, negative_slope=slope)


def MLP(channels, activation=None, bn_momentum=0.1, bias=True):
    """[Linear -> FastBatchNorm1d -> LeakyReLU(0.2)] per layer (base_modules.py:38-48)."""
    layers = []
    for i in range(1, len(channels)):
        act = activation if activation is not None else nn.LeakyReLU(0.2, inplace=True)
        layers.append(MLPLayer(nn.Linear(channels[i - 1], channels[i], bias=bias),
                               FastBatchNorm1d(channels[i], momentum=bn_momentum), act))
    return nn.Sequential(*layers)
