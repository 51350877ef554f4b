"""Image-only (No3D) segmentation models: No3DEncoder (applications/multimodal/no3d.py:14-130) and
the No3D model family (models/segmentation/multimodal/no3d.py:18-170).

The trainer around them (BaseModel, the Hydra factory) is not part of this package: the classes are
plain nn.Modules built from already-built modules, with the reference's state-dict names
(`backbone.down_modules.*`, `backbone.mlp.*`, `head.0.*`), so a reference checkpoint loads with
strict=True.  On CUDA the hot paths are this library's kernels:

  * the heads run on ops.linear (the per-pixel head reads a channels-last feature map in place);
  * eval-time propagation to unseen points uses mapping.knn_query with k = 1 (the reference's
    KeOps brute-force argmin, no3d.py:105-125): same squared distance, ties to the lowest index in
    seen order;
  * the loss is ops.csr_nll_loss, point-level on `output` or view-level on the modality's
    `last_view_x_mod` through `last_view_csr_idx` (no3d.py:141-154), without the [V] target and
    [V, K] log-prob tensors.

One deliberate difference: with seen points but no unseen point, the propagation is skipped (the
reference calls KeOps on an empty query set).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from ...core.common_modules import MLP
from ...core.multimodal.mapping import knn_query

IGNORE_LABEL = -1

__all__ = ["No3DEncoder", "No3D", "No3DFeatureFusion", "No3DLogitFusion", "No3DImageFeatureFusion",
           "No3DImageLogitFusion", "No3DOutput", "IGNORE_LABEL"]


class No3DOutput:
    """Attribute holder returned by No3DEncoder (the reference's torch_geometric Batch, :107-120):
    x, pos, seen, and one entry per modality, also reachable as out[m]."""

    def __init__(self, **kwargs):
        self.__dict__.update(kwargs)

    def __getitem__(self, key):
        return getattr(self, key)

    def __setitem__(self, key, value):
        setattr(self, key, value)

    @property
    def keys(self):
        return list(self.__dict__)


def _linear_head(x, lin):
    """nn.Linear `lin` applied to the rows of x [rows, C] on ops.linear."""
    if x.shape[0] == 0:
        return x.new_empty((0, lin.out_features))
    z = ops.linear(x, lin.weight)
    return z + lin.bias if lin.bias is not None else z


class No3DEncoder(nn.Module):
    """A stack of MultimodalBlockDown modules without 3D convolutions (applications/multimodal/no3d.py).

    down_modules: list of MultimodalBlockDown; the 3D features x_3d may be None (the modality
    branches then produce them).  output_nc: optional head MLP([default_output_nc, output_nc],
    ReLU, bias=False) applied to the point features and to every modality's last_view_x_mod
    (:118-124).  default_output_nc: the branches' output width; when None it is read from the last
    down module's branches (`out_channels`)."""

    def __init__(self, down_modules, output_nc=None, default_output_nc=None):
        super().__init__()
        self.down_modules = nn.ModuleList(down_modules)
        self._modalities = []
        for m in self.down_modules:
            for mod in m.modalities:
                if mod not in self._modalities:
                    self._modalities.append(mod)
        assert len(self._modalities) > 0, "No3DEncoder should carry at least one non-3D modality."
        if default_output_nc is None and len(self.down_modules) > 0:
            last = self.down_modules[-1]
            ncs = [getattr(last, mod)._out_channels for mod in last.modalities]
            ncs = [n for n in ncs if n is not None]
            assert all(n == ncs[0] for n in ncs), \
                f"Expected all modality branches outputs to have the same feature size but got {ncs} sizes instead."
            default_output_nc = ncs[0] if ncs else None
        self._output_nc = default_output_nc
        self._has_mlp_head = output_nc is not None
        if self._has_mlp_head:
            if default_output_nc is None:
                raise ValueError("No3DEncoder(output_nc=...) needs default_output_nc, the branches' output width")
            self._output_nc = output_nc
            self.mlp = MLP([default_output_nc, output_nc], activation=nn.ReLU(), bias=False)

    @property
    def modalities(self):
        return self._modalities

    @property
    def has_mlp_head(self):
        return self._has_mlp_head

    @property
    def output_nc(self):
        return self._output_nc

    def forward(self, data):
        """data: an object with `pos` [N, 3], `modalities` {name: ImageData} and optionally `x` [N, C]
        (3D features, None for image-only models).  Returns a No3DOutput with x [N, output_nc],
        pos, seen [N] bool (None if no branch ran) and the modality data under its name (:80-130)."""
        mm_data_dict = {'x_3d': getattr(data, 'x', None), 'x_seen': None, 'modalities': data.modalities}
        for block in self.down_modules:
            mm_data_dict = block(mm_data_dict)
        out = No3DOutput(x=mm_data_dict['x_3d'], pos=data.pos, seen=mm_data_dict['x_seen'])
        for m in self.modalities:
            out[m] = mm_data_dict['modalities'][m]
        if self.has_mlp_head:
            out.x = self.mlp(out.x)
            for m in self.modalities:
                if getattr(out[m], 'last_view_x_mod', None) is not None:
                    out[m].last_view_x_mod = self.mlp(out[m].last_view_x_mod)
        return out


class No3D(nn.Module):
    """Segmentation model on a No3DEncoder (models/segmentation/multimodal/no3d.py:18-154).

    Use the subclasses.  set_input(data) takes `data.y` [N] int64 labels (optional, may be None)
    and `data.batch`; forward() sets `output` ([N, K] log-probabilities), `loss_seg` (when labels
    are given), and `pred` / `feat` on every setting of `data.modalities[m]`:
      * _HAS_HEAD: head = nn.Sequential(nn.Linear(backbone.output_nc, num_classes)); `pred` is the
        head applied to every pixel of the feature map, `feat` the map itself;
      * otherwise the features are the logits and `pred` is the feature map.
    Training: labels of unseen points are set to -1 in place.  Eval: every unseen row of `output`
    becomes the row of its nearest seen point; with no seen point every label becomes -1 (the loss
    is then NaN).  With _MODALITY_VIEW_LOSS the loss is taken on the modality's view-level logits
    through last_view_csr_idx (its UnimodalBranch needs keep_last_view=True), otherwise on `output`.
    """

    _MODALITY_VIEW_LOSS = None

    def __init__(self, backbone, num_classes=None):
        if not hasattr(self, '_HAS_HEAD'):
            raise NotImplementedError("No3D is abstract: use one of its subclasses")
        super().__init__()
        self.backbone = backbone
        self._modalities = backbone.modalities
        if self._HAS_HEAD:
            if num_classes is None:
                raise ValueError(f"{self.__class__.__name__} needs num_classes for its head")
            self.head = nn.Sequential(nn.Linear(self.backbone.output_nc, num_classes))
        self.loss_names = ["loss_seg"]
        if self._MODALITY_VIEW_LOSS is not None:
            assert self._MODALITY_VIEW_LOSS in self._modalities, \
                f"Cannot set modality loss for '{self._MODALITY_VIEW_LOSS}'. Expected one of {self._modalities}."
        self.input, self.labels, self.batch_idx = None, None, None
        self.output, self.loss_seg = None, None

    @property
    def modalities(self):
        return self._modalities

    def set_input(self, data, device=None):
        self.input = data
        batch = getattr(data, 'batch', None)
        self.batch_idx = batch.squeeze() if batch is not None else None
        y = getattr(data, 'y', None)
        self.labels = (y.to(device) if device is not None else y) if y is not None else None

    def _head(self, x):
        return _linear_head(x, self.head[0])

    def _pixel_head(self, f_map):
        """head on every pixel of a [B, C, H, W] map -> [B, K, H, W] (no3d.py:89-96).  A channels-last
        map is read in place as [B*H*W, C] rows; the result is returned channels-last."""
        B, C, H, W = f_map.shape
        rows = f_map.permute(0, 2, 3, 1).reshape(-1, C)
        z = self._head(rows)
        return z.view(B, H, W, z.shape[1]).permute(0, 3, 1, 2)

    def forward(self, *args, **kwargs):
        data = self.backbone(self.input)
        features = data.x
        seen_mask = data.seen
        if seen_mask is None:
            seen_mask = torch.zeros(features.shape[0], dtype=torch.bool, device=features.device)

        for m in self.modalities:
            for i in range(self.input.modalities[m].num_settings):
                if self._HAS_HEAD:
                    self.input.modalities[m][i].pred = self._pixel_head(data[m][i].x)
                    self.input.modalities[m][i].feat = data[m][i].x
                else:
                    self.input.modalities[m][i].pred = data[m][i].x

        logits = self._head(features) if self._HAS_HEAD else features
        output = F.log_softmax(logits, dim=-1)

        if not self.training:
            seen_idx = torch.nonzero(seen_mask).squeeze(1)
            if seen_idx.numel() > 0:
                unseen_idx = torch.nonzero(~seen_mask).squeeze(1)
                if unseen_idx.numel() > 0:
                    # nearest seen point of every unseen point (no3d.py:105-125)
                    pos = data.pos.to(features.device)
                    nn_idx = knn_query(pos[unseen_idx], pos[seen_idx], 1).squeeze(1)
                    output = output.index_put((unseen_idx,), output[seen_idx[nn_idx]])
            elif self.labels is not None:
                self.labels[~seen_mask] = IGNORE_LABEL
        elif self.labels is not None:
            self.labels[~seen_mask] = IGNORE_LABEL
        self.output = output

        if self.labels is not None:
            if self._MODALITY_VIEW_LOSS is None:
                self.loss_seg = ops.csr_nll_loss(self.output, self.labels, None, ignore_index=IGNORE_LABEL)
            else:
                mod = data[self._MODALITY_VIEW_LOSS]
                view_features = mod.last_view_x_mod
                view_logits = self._head(view_features) if self._HAS_HEAD else view_features
                self.loss_seg = ops.csr_nll_loss(view_logits, self.labels, mod.last_view_csr_idx,
                                                 ignore_index=IGNORE_LABEL)
        return self.output

    def backward(self):
        self.loss_seg.backward()


class No3DFeatureFusion(No3D):
    _HAS_HEAD = True


class No3DLogitFusion(No3D):
    _HAS_HEAD = False


class No3DImageFeatureFusion(No3D):
    _HAS_HEAD = True
    _MODALITY_VIEW_LOSS = 'image'


class No3DImageLogitFusion(No3D):
    _HAS_HEAD = False
    _MODALITY_VIEW_LOSS = 'image'
