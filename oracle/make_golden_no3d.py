"""Generate the No3D model fixtures by EXECUTING THE REFERENCE (oracle; test infrastructure).

Run in the build container only (needs the reference checkout, see oracle/ref_loader.py):
    PYTORCH_JIT=0 python -m oracle.make_golden_no3d
writes tests/golden/no3d_{main,ties,noseen,allseen}.npz.

The reference's `No3D.forward` (models/segmentation/multimodal/no3d.py:73-157) and
`No3DEncoder.forward` (applications/multimodal/no3d.py:79-130) run unchanged on the reference's
MultimodalBlockDown / UnimodalBranch / pools / ImageData (CPU, torch_scatter stand-in), with
stand-ins for what the trainer provides: BaseModel (an nn.Module with `device` and `modalities`),
IGNORE_LABEL = -1, torch_geometric's Batch (an attribute holder) and KeOps' LazyTensor.  The
LazyTensor stand-in is dense and gains `argmin(dim)` (torch.argmin: the first minimum, i.e. ties to
the lowest index in seen order), so the nearest-seen-point search is restated, not executed, as for
the Biasutti fixtures.  The head MLP is the reference's MLP, loaded by path.

Per sample and per class (No3DFeatureFusion, No3DLogitFusion, No3DImageFeatureFusion,
No3DImageLogitFusion) and mode (train / eval): the model's state dict (`sd/<cls>/...`) and
`<cls>/<mode>/{output, loss, labels}` and `<cls>/pred<i>` (the pixel head, the same in both modes).
"""
import os
import sys

os.environ.setdefault("PYTORCH_JIT", "0")

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch import nn  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle.make_golden import save  # noqa: E402

CLASSES = ("No3DFeatureFusion", "No3DLogitFusion", "No3DImageFeatureFusion", "No3DImageLogitFusion")
NUM_CLASSES = 5
C_FEAT = 8          # feature-map channels of the *FeatureFusion samples (head: Linear(8, 5))


class DenseArgminLazyTensor:
    """Dense stand-in for the pykeops LazyTensor operations of no3d.py:116-120: broadcasting `-`,
    `** 2`, `.sum(dim=2)` and `.argmin(dim=1)`; KeOps returns the argmin as an [M, 1] tensor."""

    def __init__(self, t):
        self.t = t

    def __sub__(self, other):
        return DenseArgminLazyTensor(self.t - other.t)

    def __pow__(self, p):
        return DenseArgminLazyTensor(self.t ** p)

    def sum(self, dim):
        return DenseArgminLazyTensor(self.t.sum(dim=dim))

    def argmin(self, dim):
        return torch.argmin(self.t, dim=dim, keepdim=True)


class Batch:
    """torch_geometric.data.Batch stand-in: an attribute holder with item access and `keys`."""

    def __init__(self, **kwargs):
        self.__dict__.update(kwargs)

    def __getitem__(self, key):
        return getattr(self, key)

    def __setitem__(self, key, value):
        setattr(self, key, value)

    @property
    def keys(self):
        return list(self.__dict__)


class MMData:
    """The MMData fields No3D / No3DEncoder read: x, pos, y, batch, modalities."""

    def __init__(self, **kwargs):
        self.__dict__.update(kwargs)

    def to(self, device):
        return self


def load_no3d():
    """The reference's No3DEncoder and No3D classes, loaded by path with the stand-ins above."""
    ns = ref_loader.load_reference()
    if hasattr(ns, "no3d"):
        return ns
    st = ref_loader._stub
    bb = st("torch_points3d.models.base_architectures.backbone")
    bb.BackboneBasedModel = nn.Module
    st("torch_points3d.models")
    st("torch_points3d.models.base_architectures")
    st("torch_points3d.applications")
    st("torch_points3d.applications.utils").extract_output_nc = None
    st("torch_points3d.core.multimodal.data").MMData = MMData
    st("torch_geometric")
    st("torch_geometric.data").Batch = Batch

    class BaseModel(nn.Module):
        def __init__(self, option=None):
            super().__init__()

        @property
        def device(self):
            return torch.device("cpu")

        @property
        def modalities(self):
            return self._modalities

    st("torch_points3d.models.base_model").BaseModel = BaseModel
    st("torch_points3d.datasets")
    st("torch_points3d.datasets.segmentation").IGNORE_LABEL = -1
    sys.modules["pykeops.torch"].LazyTensor = DenseArgminLazyTensor
    st("torch_points3d.applications.multimodal")
    ns.no3d_encoder = ref_loader._load("torch_points3d.applications.multimodal.no3d",
                                       "torch_points3d/applications/multimodal/no3d.py")
    st("torch_points3d.models.segmentation")
    st("torch_points3d.models.segmentation.multimodal")
    ns.no3d = ref_loader._load("torch_points3d.models.segmentation.multimodal.no3d",
                               "torch_points3d/models/segmentation/multimodal/no3d.py")
    ns.BaseModel = BaseModel
    return ns


def make_encoder(ns, down_modules, output_nc, default_output_nc):
    """A reference No3DEncoder without its config-driven __init__ (BackboneBasedModel): the
    attributes its forward reads, and its own forward / _set_input."""
    E = ns.no3d_encoder.No3DEncoder

    class Encoder(nn.Module):
        forward = E.forward
        _set_input = E._set_input
        has_mlp_head = E.has_mlp_head
        output_nc = E.output_nc

        @property
        def modalities(self):
            return self._modalities

        @property
        def device(self):
            return torch.device("cpu")

    enc = Encoder()
    enc.down_modules = nn.ModuleList(down_modules)
    enc._modalities = ["image"]
    enc._output_nc = default_output_nc
    enc._has_mlp_head = output_nc is not None
    if enc._has_mlp_head:
        enc._output_nc = output_nc
        enc.mlp = ns.base_modules.MLP([default_output_nc, output_nc], activation=nn.ReLU(), bias=False)
    return enc


def make_model(ns, cls_name, enc):
    cls = getattr(ns.no3d, cls_name)
    model = cls.__new__(cls)
    nn.Module.__init__(model)
    model.backbone = enc
    model._modalities = enc._modalities
    if cls._HAS_HEAD:
        model.head = nn.Sequential(nn.Linear(enc.output_nc, NUM_CLASSES))
    model.loss_names = ["loss_seg"]
    return model


def sample_inputs(kind, gen):
    """pos [N,3], labels [N], per setting (W, H, n_img, pid, iid, pix, feat).  `seen_region` points
    get views; the others are unseen (a whole region, as surfaces outside every camera)."""
    if kind == "ties":
        # seen points on an integer lattice with duplicates; unseen points at lattice midpoints,
        # equidistant from two (or more) seen points
        a = torch.arange(6, dtype=torch.float32)
        lat = torch.stack(torch.meshgrid(a, a, torch.zeros(1), indexing="ij"), -1).reshape(-1, 3)
        seen_pos = torch.cat([lat, lat[::3]])                        # every third lattice point twice
        unseen_pos = lat[:-1] + torch.tensor([0.5, 0.0, 0.0])
        unseen_pos = torch.cat([unseen_pos, lat[:10] + torch.tensor([0.5, 0.5, 0.0])])
        pos = torch.cat([seen_pos, unseen_pos])
        seen_cand = torch.zeros(pos.shape[0], dtype=torch.bool)
        seen_cand[:seen_pos.shape[0]] = True
        perm = torch.randperm(pos.shape[0], generator=gen)
        pos, seen_cand = pos[perm], seen_cand[perm]
    else:
        n = 300
        pos = torch.rand(n, 3, generator=gen) * torch.tensor([4.0, 3.0, 1.5])
        if kind == "allseen":
            seen_cand = torch.ones(n, dtype=torch.bool)
        else:
            seen_cand = (pos[:, 0] < 2.2) | (torch.rand(n, generator=gen) < 0.05)
    n = pos.shape[0]
    labels = torch.randint(0, NUM_CLASSES, (n,), generator=gen)
    labels[torch.rand(n, generator=gen) < 0.1] = -1
    settings = []
    if kind == "noseen":
        return pos, labels, settings
    for (W, H, n_img) in ((16, 12, 3), (12, 12, 2)):
        counts = torch.poisson(torch.full((n,), 1.8), generator=gen).clamp(0, n_img).long()
        counts[~seen_cand] = 0
        if kind in ("allseen", "ties"):
            counts[seen_cand] = counts[seen_cand].clamp(min=1)
        pid = torch.arange(n).repeat_interleave(counts)
        iid = torch.cat([torch.randperm(n_img, generator=gen)[:int(c)] for c in counts]) if pid.numel() else pid
        pix = torch.stack([torch.randint(0, W, (pid.numel(),), generator=gen),
                           torch.randint(0, H, (pid.numel(),), generator=gen)], 1).short()
        feat = torch.rand(pid.numel(), 4, generator=gen)
        settings.append(dict(W=W, H=H, n_img=n_img, pid=pid, iid=iid, pix=pix, feat=feat))
    return pos, labels, settings


def run_reference(ns, cls_name, mode, pos, labels, settings, maps, x3d, sd):
    """maps: one [n_img, C, H, W] feature map per setting (image-only input); or no setting at all
    and x3d [N, C] 3D features (no point is seen: the branch passes x3d through, modules.py:317-365)."""
    I, P, M = ns.image, ns.pooling, ns.modules
    ims = []
    for st, x in zip(settings, maps):
        im = I.SameSettingImageData(path=np.array([f"img_{i}" for i in range(st["n_img"])]),
                                    pos=torch.zeros(st["n_img"], 3), opk=torch.zeros(st["n_img"], 3),
                                    ref_size=(st["W"], st["H"]), proj_upscale=1, downscale=1)
        im.mappings = I.ImageMapping.from_dense(st["pid"], st["iid"], st["pix"], st["feat"], num_points=pos.shape[0])
        im.x = x.clone()
        ims.append(im)
    mod = I.ImageData(ims)
    c = maps[0].shape[1] if maps else x3d.shape[1]
    branch = M.UnimodalBranch(None, P.BimodalCSRPool(mode="max"), P.BimodalCSRPool(mode="mean"),
                              ns.fusion.BimodalFusion("residual"), keep_last_view=True, out_channels=c)
    block = M.MultimodalBlockDown(None, None, image=branch)
    # the logit classes carry the optional encoder head MLP([5, 5]) when there are views to apply it to
    mlp = "Logit" in cls_name and maps
    enc = make_encoder(ns, [block], NUM_CLASSES if mlp else None, c)
    model = make_model(ns, cls_name, enc)
    if sd is not None:
        model.load_state_dict(sd, strict=True)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    model.train(mode == "train")
    data = MMData(x=x3d, pos=pos.clone(), y=labels.clone(), batch=None, modalities={"image": mod})
    with torch.no_grad():
        model.set_input(data, "cpu")
        model.forward()
    out = {"output": model.output, "loss": model.loss_seg.reshape(()), "labels": model.labels}
    for i in range(len(ims)):
        if model._HAS_HEAD:
            assert mod[i].feat is mod[i].x
            out[f"pred{i}"] = mod[i].pred            # the head on every pixel
        else:
            assert mod[i].pred is mod[i].x           # the logit classes: the map itself
    return out, sd


def make_sample(ns, kind, seed):
    gen = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    pos, labels, settings = sample_inputs(kind, gen)
    arrays = {"pos": pos, "labels": labels}
    for s, st in enumerate(settings):
        for k in ("pid", "iid", "pix", "feat"):
            arrays[f"s{s}_{k}"] = st[k]
        arrays[f"s{s}_size"] = np.array([st["W"], st["H"], st["n_img"]])
    seen = torch.zeros(pos.shape[0], dtype=torch.bool)
    for st in settings:
        seen[st["pid"]] = True
    arrays["seen"] = seen
    # with no view at all the reference's view-loss classes have no last_view_x_mod to read
    classes = CLASSES if settings else ("No3DFeatureFusion", "No3DLogitFusion")
    for cls_name in classes:
        c = NUM_CLASSES if "Logit" in cls_name else C_FEAT
        maps = [torch.randn(st["n_img"], c, st["H"], st["W"], generator=gen) for st in settings]
        for s, x in enumerate(maps):
            arrays[f"{cls_name}/map{s}"] = x
        x3d = None
        if not settings:
            x3d = torch.randn(pos.shape[0], c, generator=gen)
            arrays[f"{cls_name}/x3d"] = x3d
        sd = None
        for mode in ("train", "eval"):
            out, sd = run_reference(ns, cls_name, mode, pos, labels, settings, maps, x3d, sd)
            if mode == "train":
                for k, v in sd.items():
                    arrays[f"sd/{cls_name}/{k}"] = v
            for k, v in out.items():
                if k.startswith("pred") and mode == "eval":
                    assert torch.equal(v, arrays[f"{cls_name}/{k}"])
                    continue
                arrays[f"{cls_name}/{k}" if k.startswith("pred") else f"{cls_name}/{mode}/{k}"] = v
    save(f"no3d_{kind}", **arrays)


def main():
    ns = load_no3d()
    for kind, seed in (("main", 71), ("ties", 72), ("noseen", 73), ("allseen", 74)):
        make_sample(ns, kind, seed)


if __name__ == "__main__":
    main()
