"""Dense stand-ins for the caller-built parts of the sparse-conv fusion models (TEST INFRASTRUCTURE ONLY): the
sparse 3D UNet, the No3D encoder and the sparse ResBlock used as `late_conv`.  Shared by
oracle/make_golden_sparseconv3d.py, which runs the reference's model classes on them, and by
tests/test_gpu_sparseconv3d.py, which runs this package's classes on the same modules and state dicts.

Protocols kept (models/segmentation/multimodal/sparseconv3d.py:114-137):
  * the 3D backbone is called on `input.data`, returns an object with `.x`, and exposes `last_sparse_tensor`
    whose `.F` the model overwrites with the fused features;
  * the No3D backbone is called on the whole input and reads its 3D features from `input.x` (= `input.data.x`,
    which the model swaps for the 3D backbone's output), so a missed swap changes the result;
  * late_conv takes the sparse tensor and returns one with `.F`.
"""
import torch
from torch import nn


class Data:
    """torch_geometric Data stand-in: an attribute holder."""

    def __init__(self, **kwargs):
        self.__dict__.update(kwargs)


class MMData:
    """MMData stand-in: `data` (x, y, batch, pos) and `modalities`; x / y / batch / pos read through to `data`."""

    def __init__(self, data, modalities=None):
        self.data = data
        self.modalities = modalities if modalities is not None else {}

    @property
    def x(self):
        return self.data.x

    @x.setter
    def x(self, v):
        self.data.x = v

    @property
    def y(self):
        return self.data.y

    @property
    def batch(self):
        return self.data.batch

    @property
    def pos(self):
        return self.data.pos


class SparseLike:
    def __init__(self, F):
        self.F = F


class Output:
    def __init__(self, x):
        self.x = x


class DenseBackbone3D(nn.Module):
    """x -> relu(lin(x)); `last_sparse_tensor.F` holds the output."""

    def __init__(self, c_in, c_out):
        super().__init__()
        self.lin = nn.Linear(c_in, c_out)
        self.output_nc = c_out
        self._modalities = []
        self.last_sparse_tensor = None

    def forward(self, data):
        f = torch.relu(self.lin(data.x))
        self.last_sparse_tensor = SparseLike(f)
        return Output(f)


class DenseNo3D(nn.Module):
    """input.x (the 3D features swapped in by the model) -> tanh(lin(.)); `modalities` = ['image']."""

    def __init__(self, c_in, c_out):
        super().__init__()
        self.lin = nn.Linear(c_in, c_out)
        self.output_nc = c_out
        self.modalities = ["image"]

    def forward(self, mm):
        return Output(torch.tanh(self.lin(mm.x)))


class DenseLateConv(nn.Module):
    """sparse tensor -> SparseLike(relu(lin(F))).  The reference builds late_conv for backbone_3d.output_nc +
    backbone_no3d.output_nc input channels whatever the fusion mode, while 'residual' fusion hands it
    output_nc channels; a narrower F is zero-padded on the right so that every mode runs."""

    def __init__(self, c_in, c_out=96):
        super().__init__()
        self.lin = nn.Linear(c_in, c_out)

    def forward(self, st):
        f = st.F
        if f.shape[1] < self.lin.in_features:
            f = torch.nn.functional.pad(f, (0, self.lin.in_features - f.shape[1]))
        return SparseLike(torch.relu(self.lin(f)))
