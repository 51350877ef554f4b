"""Sparse-conv segmentation models: APIModel (models/segmentation/sparseconv3d.py:15-63) and the late fusion
models LateFeatureFusion and LateLogitFusion (models/segmentation/multimodal/sparseconv3d.py:12-226).

The trainer around them (BaseModel, the Hydra factory) and the sparse 3D backbone are not part of this package:
the classes are plain nn.Modules built from already-built modules, with the reference's state-dict names
(`backbone.*`, `head.0.*`; `backbone_3d.*`, `backbone_no3d.*`, `late_conv.*`, `head.*`, `head_no3d.0.*`,
`head_3d.0.*`), so a reference checkpoint loads with strict=True.  On CUDA the hot paths are this library's
kernels:

  * the heads run on ops.linear;
  * the cross-entropy is ops.csr_nll_loss on the logits (log_softmax only produces `output`), with the class
    weights when given;
  * the Lovász term is ops.lovasz_softmax(output, labels, log_probs=True): the reference's
    lovasz_softmax(output.exp(), labels, ignore=-1), exp taken in the kernel.

Reproduced quirks: LateFeatureFusion adds the auxiliary no3d / 3D NLL terms once whatever the loss options
(:141-152), then again under use_cross_entropy (:166-179), so with cross-entropy on they count twice; those
auxiliary terms are unweighted, and so is its main cross-entropy (the reference reads a `_weight_classes` its
__init__ never sets, unless the caller passes weight_classes here).  'residual' fusion hands late_conv
output_nc channels although the reference builds late_conv for the sum of both backbones' widths.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from .no3d import IGNORE_LABEL, _linear_head

__all__ = ["APIModel", "LateFeatureFusion", "LateLogitFusion"]


class _SparseConvModel(nn.Module):
    """set_input / backward / loss bookkeeping shared by the three classes (sparseconv3d.py:34-63)."""

    def _init_losses(self, use_cross_entropy, use_lovasz):
        self._use_cross_entropy = use_cross_entropy
        self._use_lovasz = use_lovasz
        assert self._use_cross_entropy or self._use_lovasz, \
            "Choose at least one between Cross-Entropy loss and Lovasz loss."
        self.input, self.labels, self.batch_idx = None, None, None
        self.output, self.loss_seg = None, None

    @property
    def modalities(self):
        return self._modalities

    def set_input(self, data, device=None):
        batch = getattr(data, 'batch', None)
        self.batch_idx = batch.squeeze() if batch is not None else None
        self.input = data
        y = getattr(data, 'y', None)
        self.labels = (y.to(device) if device is not None else y) if y is not None else None

    # the tracker interface of the reference's BaseModel (metrics/*_tracker.py read these)
    def get_input(self):
        return self.input

    def get_output(self):
        return self.output

    def get_labels(self):
        return self.labels

    @property
    def is_multimodal(self):
        return bool(self._modalities)

    def _nll(self, logits, weight=None):
        return ops.csr_nll_loss(logits, self.labels, None, ignore_index=IGNORE_LABEL, weight=weight)

    def _lovasz(self, log_probs):
        return ops.lovasz_softmax(log_probs, self.labels, ignore=IGNORE_LABEL, log_probs=True)

    def backward(self):
        self.loss_seg.backward()


class APIModel(_SparseConvModel):
    """Sparse UNet + linear head (models/segmentation/sparseconv3d.py:15-63): the early / intermediate fusion
    models, whose `backbone` (the caller's sparse UNet, possibly with MultimodalBlockDown down modules) does the
    fusion.  forward() sets `output` ([N, K] log-probabilities) and, with labels, `loss_seg` and
    `loss_cross_entropy` / `loss_lovasz`.  weight_classes: optional [K] float32 class weights of the
    cross-entropy (the dataset's weight_classes)."""

    def __init__(self, backbone, num_classes, use_cross_entropy=True, use_lovasz=False, weight_classes=None):
        super().__init__()
        self._weight_classes = weight_classes
        self.backbone = backbone
        self._modalities = getattr(backbone, '_modalities', [])
        self.head = nn.Sequential(nn.Linear(backbone.output_nc, num_classes))
        self._init_losses(use_cross_entropy, use_lovasz)
        self.loss_names = ['loss_seg'] + use_cross_entropy * ['loss_cross_entropy'] + use_lovasz * ['loss_lovasz']

    def forward(self, *args, **kwargs):
        features = self.backbone(self.input).x
        logits = _linear_head(features, self.head[0])
        self.output = F.log_softmax(logits, dim=-1)
        if self._weight_classes is not None:
            self._weight_classes = self._weight_classes.to(logits.device)
        if self.labels is not None:
            self.loss_seg = 0
            if self._use_cross_entropy:
                self.loss_cross_entropy = self._nll(logits, self._weight_classes)
                self.loss_seg += self.loss_cross_entropy
            if self._use_lovasz:
                self.loss_lovasz = self._lovasz(self.output)
                self.loss_seg += self.loss_lovasz
        return self.output


class LateFeatureFusion(_SparseConvModel):
    """A sparse 3D backbone and a No3DEncoder with late feature fusion
    (models/segmentation/multimodal/sparseconv3d.py:12-182).

    backbone_3d: called on `input.data`, returns `.x` [N, C3] and exposes `last_sparse_tensor`, whose `.F` is
    set to the fused features before late_conv runs on it (late_conv returns a sparse tensor with `.F`
    [N, 96]).  backbone_no3d: this package's No3DEncoder, called on the whole input while `input.data.x` holds
    the 3D features (restored afterwards).  mode: 'residual' (a + b), 'concatenation' (cat(a, b)) or 'both'
    (cat(a, a + b)).  loss_no3d / loss_3d add auxiliary heads on each backbone's features."""

    MODES = ['residual', 'concatenation', 'both']

    def __init__(self, backbone_3d, backbone_no3d, late_conv, num_classes, mode='residual', loss_no3d=False,
                 loss_3d=False, use_cross_entropy=True, use_lovasz=False, weight_classes=None):
        super().__init__()
        self.backbone_3d = backbone_3d
        self.backbone_no3d = backbone_no3d
        self._modalities = backbone_no3d.modalities
        self.mode = mode if mode is not None else 'residual'
        if self.mode in ('residual', 'both'):
            assert backbone_3d.output_nc == backbone_no3d.output_nc, \
                f"Backbones output dimensions must be the same. Received " \
                f"backbone_3d.output_nc={backbone_3d.output_nc} and " \
                f"backbone_no3d.output_nc={backbone_no3d.output_nc} instead."
        elif self.mode != 'concatenation':
            raise NotImplementedError(f"Unknown fusion mode='{self.mode}'. Please choose among supported modes: "
                                      f"{self.MODES}.")
        self.late_conv = late_conv
        self.head = nn.Linear(96, num_classes)
        self.head_no3d = nn.Sequential(nn.Linear(backbone_no3d.output_nc, num_classes)) if loss_no3d else None
        self.head_3d = nn.Sequential(nn.Linear(backbone_3d.output_nc, num_classes)) if loss_3d else None
        self._weight_classes = weight_classes
        self._init_losses(use_cross_entropy, use_lovasz)
        ce, lov = use_cross_entropy, use_lovasz
        self.loss_names = ['loss_seg'] + ce * ['loss_cross_entropy'] + lov * ['loss_lovasz'] \
            + (ce and loss_no3d) * ['loss_cross_entropy_no3d'] + (ce and loss_3d) * ['loss_cross_entropy_3d'] \
            + (lov and loss_no3d) * ['loss_lovasz_no3d'] + (lov and loss_3d) * ['loss_lovasz_3d']

    def fusion(self, a, b):
        if self.mode == 'residual':
            return a + b
        if self.mode == 'concatenation':
            return torch.cat((a, b), dim=-1)
        return torch.cat((a, a + b), dim=-1)

    def forward(self, *args, **kwargs):
        features_3d = self.backbone_3d(self.input.data).x

        # the No3D backbone reads the 3D features from the input: swap them in, restore the input afterwards
        input_x_backup = self.input.data.x
        self.input.data.x = features_3d
        try:
            features_no3d = self.backbone_no3d(self.input).x
        finally:
            self.input.data.x = input_x_backup

        sparse_features = self.backbone_3d.last_sparse_tensor
        sparse_features.F = self.fusion(features_3d, features_no3d)
        features = self.late_conv(sparse_features).F

        logits = _linear_head(features, self.head)
        self.output = F.log_softmax(logits, dim=-1)
        if self._weight_classes is not None:
            self._weight_classes = self._weight_classes.to(logits.device)

        if self.labels is not None:
            logits_no3d = _linear_head(features_no3d, self.head_no3d[0]) if self.head_no3d else None
            logits_3d = _linear_head(features_3d, self.head_3d[0]) if self.head_3d else None
            self.loss_seg = 0
            # auxiliary NLL terms, added whatever the loss options (:141-152)
            if logits_no3d is not None:
                self.loss_seg += self._nll(logits_no3d)
            if logits_3d is not None:
                self.loss_seg += self._nll(logits_3d)
            if self._use_cross_entropy:
                self.loss_cross_entropy = self._nll(logits, self._weight_classes)
                self.loss_seg += self.loss_cross_entropy
            if self._use_lovasz:
                self.loss_lovasz = self._lovasz(self.output)
                self.loss_seg += self.loss_lovasz
            # and again under the loss options (:162-181)
            for name, aux in (('no3d', logits_no3d), ('3d', logits_3d)):
                if aux is None:
                    continue
                if self._use_cross_entropy:
                    loss = self._nll(aux)
                    setattr(self, f'loss_cross_entropy_{name}', loss)
                    self.loss_seg += loss
                if self._use_lovasz:
                    loss = self._lovasz(F.log_softmax(aux, dim=-1))
                    setattr(self, f'loss_lovasz_{name}', loss)
                    self.loss_seg += loss
        return self.output


class LateLogitFusion(_SparseConvModel):
    """A sparse 3D backbone and a No3DEncoder whose outputs are logits, summed
    (models/segmentation/multimodal/sparseconv3d.py:185-226).  backbone_3d is called on `input.data`,
    backbone_no3d (its head set in the encoder, e.g. `last_conv`) on the whole input; head_3d maps the 3D
    features to logits.  The loss is the NLL of the summed logits."""

    def __init__(self, backbone_3d, backbone_no3d, num_classes):
        super().__init__()
        self.backbone_3d = backbone_3d
        self.backbone_no3d = backbone_no3d
        self._modalities = backbone_no3d.modalities
        self.head_3d = nn.Sequential(nn.Linear(backbone_3d.output_nc, num_classes))
        self._init_losses(True, False)
        self.loss_names = ['loss_seg']

    def forward(self, *args, **kwargs):
        features_3d = self.backbone_3d(self.input.data).x
        logits_3d = _linear_head(features_3d, self.head_3d[0])
        logits_no3d = self.backbone_no3d(self.input).x
        logits = logits_3d + logits_no3d
        self.output = F.log_softmax(logits, dim=-1)
        if self.labels is not None:
            self.loss_seg = self._nll(logits)
        return self.output
