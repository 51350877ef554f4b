"""Generate the Lovász-softmax and sparse-conv fusion model fixtures by EXECUTING THE REFERENCE (oracle; test
infrastructure).

Run in the build container only (needs the reference checkout, see oracle/ref_loader.py):
    python -m oracle.make_golden_sparseconv3d
writes tests/golden/lovasz_{tiefree,ties,ignored,absent,all,list}.npz and tests/golden/sparseconv3d_models.npz.

Lovász: the reference's metrics/lovasz_loss.py, loaded by path, runs lovasz_softmax(probas, labels, classes,
ignore=-1) on fp32 CPU tensors; the fixture holds the inputs, the loss and d loss / d probas (autograd).  CPU
torch.sort is unstable, so on tied inputs only the loss is meaningful.

Models: models/segmentation/sparseconv3d.py (APIModel) and models/segmentation/multimodal/sparseconv3d.py
(LateFeatureFusion, LateLogitFusion) run their own __init__, set_input, forward and backward, with stand-ins
for what they import but the fixtures do not exercise: BaseModel (an nn.Module with `device`), IGNORE_LABEL =
-1, resolve_model (no-op), and factories in place of SparseConv3d / No3DEncoder / ResBlock that return the
dense modules of oracle/sparseconv3d_fakes.py.  Per case: the state dict (`<case>/sd/...`), `output`, every
`loss_*` of `loss_names` and the gradients of the head parameters (`<case>/grad/...`).
"""
import os
import sys

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle import sparseconv3d_fakes as fk  # noqa: E402
from oracle.make_golden import save  # noqa: E402

NUM_CLASSES = 5
C_IN, C_3D = 6, 16
N_POINTS = 240

# (case, class, options)
MODEL_CASES = [
    ("api_ce", "APIModel", dict(use_cross_entropy=True, use_lovasz=False)),
    ("api_ce_weighted_lovasz", "APIModel", dict(use_cross_entropy=True, use_lovasz=True, weighted=True)),
    ("api_lovasz", "APIModel", dict(use_cross_entropy=False, use_lovasz=True)),
]
for _mode in ("residual", "concatenation", "both"):
    for _no3d, _3d, _ce, _lov in ((False, False, True, False), (True, True, True, True),
                                  (True, False, False, True), (False, True, True, False)):
        MODEL_CASES.append((f"late_{_mode}_{int(_no3d)}{int(_3d)}{int(_ce)}{int(_lov)}", "LateFeatureFusion",
                            dict(mode=_mode, loss_no3d=_no3d, loss_3d=_3d, use_cross_entropy=_ce, use_lovasz=_lov)))
MODEL_CASES.append(("late_logit", "LateLogitFusion", {}))


class Option(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


def load_lovasz():
    ref_loader._stub("torch_points3d")
    ref_loader._stub("torch_points3d.metrics")
    return ref_loader._load("torch_points3d.metrics.lovasz_loss", "torch_points3d/metrics/lovasz_loss.py")


def load_models():
    """The reference's APIModel, LateFeatureFusion and LateLogitFusion, loaded by path with stand-ins."""
    st = ref_loader._stub
    load_lovasz()

    class BaseModel(nn.Module):
        def __init__(self, option=None):
            super().__init__()

        @property
        def device(self):
            return torch.device("cpu")

    st("torch_points3d.models")
    st("torch_points3d.models.base_model").BaseModel = BaseModel
    st("torch_points3d.datasets")
    st("torch_points3d.datasets.segmentation").IGNORE_LABEL = -1
    st("torch_points3d.applications")
    st("torch_points3d.applications.sparseconv3d").SparseConv3d = \
        lambda arch, c_in, config=None, backend=None: fk.DenseBackbone3D(c_in, config["output_nc"])
    sp3d = st("torch_points3d.modules.SparseConv3d")
    sp3d.nn = Option(get_backend=lambda: "minkowski", Conv3d=None)
    st("torch_points3d.modules")
    st("torch_points3d.modules.SparseConv3d.modules").ResBlock = lambda c_in, c_out, conv: fk.DenseLateConv(c_in, c_out)
    st("torch_points3d.applications.multimodal")
    st("torch_points3d.applications.multimodal.no3d").No3DEncoder = \
        lambda option, model_type, dataset, modules: fk.DenseNo3D(option["c_in"], option["output_nc"])
    st("torch_points3d.utils")
    st("torch_points3d.utils.model_building_utils")
    st("torch_points3d.utils.model_building_utils.model_definition_resolver").resolve_model = lambda *a: None
    st("torch_points3d.models.segmentation")
    st("torch_points3d.models.segmentation.multimodal")
    st("torch_points3d.models.segmentation.multimodal.no3d").torch = torch
    single = ref_loader._load("torch_points3d.models.segmentation.sparseconv3d",
                              "torch_points3d/models/segmentation/sparseconv3d.py")
    multi = ref_loader._load("torch_points3d.models.segmentation.multimodal.sparseconv3d",
                             "torch_points3d/models/segmentation/multimodal/sparseconv3d.py")
    return dict(APIModel=single.APIModel, LateFeatureFusion=multi.LateFeatureFusion,
                LateLogitFusion=multi.LateLogitFusion)


# ------------------------------------------------------------------------------------------------
# Lovász
# ------------------------------------------------------------------------------------------------
def lovasz_inputs(kind, gen):
    P, K = 300, 6
    probas = torch.softmax(2 * torch.randn(P, K, generator=gen), -1)
    labels = torch.randint(0, K, (P,), generator=gen)
    classes = "present"
    if kind == "ties":
        probas = (probas * 8).round() / 8                       # few distinct values: many tied errors
    if kind in ("ignored", "ties", "absent", "all", "list"):
        labels[torch.rand(P, generator=gen) < 0.15] = -1
    if kind in ("absent", "all", "list"):
        labels[labels == 3] = 0                                 # class 3 has no point
    if kind == "all":
        classes = "all"
    if kind == "list":
        classes = [0, 2, 2, 3, 5]
    return probas.float(), labels, classes


def make_lovasz(lv):
    for kind, seed in (("tiefree", 11), ("ties", 12), ("ignored", 13), ("absent", 14), ("all", 15), ("list", 16)):
        gen = torch.Generator().manual_seed(seed)
        probas, labels, classes = lovasz_inputs(kind, gen)
        x = probas.clone().requires_grad_(True)
        loss = lv.lovasz_softmax(x, labels, classes=classes, ignore=-1)
        loss.backward()
        save(f"lovasz_{kind}", probas=probas, labels=labels, loss=loss.detach().reshape(()), grad=x.grad,
             classes=np.array(classes if isinstance(classes, list) else [], dtype=np.int64),
             classes_mode=np.array(classes if isinstance(classes, str) else "list"))


# ------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------
def make_models(classes):
    gen = torch.Generator().manual_seed(31)
    x = torch.randn(N_POINTS, C_IN, generator=gen)
    y = torch.randint(0, NUM_CLASSES, (N_POINTS,), generator=gen)
    y[torch.rand(N_POINTS, generator=gen) < 0.1] = -1
    weights = torch.rand(NUM_CLASSES, generator=gen) + 0.25
    arrays = dict(x=x, y=y, weight_classes=weights, num_classes=np.array(NUM_CLASSES), c_3d=np.array(C_3D))
    for i, (case, cls_name, opts) in enumerate(MODEL_CASES):
        torch.manual_seed(100 + i)
        opts = dict(opts)
        weighted = opts.pop("weighted", False)
        dataset = Option(num_classes=NUM_CLASSES, feature_dimension=C_IN,
                         weight_classes=weights.clone() if weighted else None)
        if cls_name == "APIModel":
            option = Option(backbone={"output_nc": C_3D}, **opts)
            data = fk.Data(x=x.clone(), y=y.clone(), batch=torch.zeros(N_POINTS, dtype=torch.long))
        else:
            no3d_nc = NUM_CLASSES if cls_name == "LateLogitFusion" else (C_3D + 4 if opts.get("mode") ==
                                                                         "concatenation" else C_3D)
            # LateLogitFusion runs backbone_no3d on the raw input; LateFeatureFusion on the 3D features
            no3d_in = C_IN if cls_name == "LateLogitFusion" else C_3D
            option = Option(backbone_3d={"output_nc": C_3D}, backbone_no3d={"output_nc": no3d_nc, "c_in": no3d_in},
                            **opts)
            data = fk.MMData(fk.Data(x=x.clone(), y=y.clone(), batch=torch.zeros(N_POINTS, dtype=torch.long)))
        model = classes[cls_name](option, "segmentation", dataset, None)
        model.set_input(data, "cpu")
        model.forward()
        model.backward()
        if cls_name != "APIModel":
            assert data.data.x is not None and torch.equal(data.data.x, x)
        arrays[f"{case}/output"] = model.output.detach()
        for name in model.loss_names:
            v = getattr(model, name)
            arrays[f"{case}/{name}"] = (v.detach() if torch.is_tensor(v) else torch.tensor(float(v))).reshape(())
        for k, v in model.state_dict().items():
            arrays[f"{case}/sd/{k}"] = v
        for k, p in model.named_parameters():
            if k.startswith("head") and p.grad is not None:
                arrays[f"{case}/grad/{k}"] = p.grad
        arrays[f"{case}/loss_names"] = np.array(model.loss_names)
    save("sparseconv3d_models", **arrays)


def main():
    make_lovasz(load_lovasz())
    make_models(load_models())


if __name__ == "__main__":
    main()
