"""Fixtures of the ImageNet and Cityscapes ResNet-18 encoders, made by EXECUTING the reference's ResNet18* and
CityscapesResNet18* wrappers (torch_points3d/modules/multimodal/modalities/image.py:959-1399), loaded by file path in
float64 on the CPU, with the installed torchvision's ResNet.

    PYTORCH_JIT=0 python -m oracle.make_golden_image_resnet18_families   # tests/golden/image_resnet18_families_*.npz

The reference module is loaded with the stubs of oracle/make_golden_image_resnet18.py.  Its constructors load the
reference's own imagenet/resnet18/resnet18.pth and cityscapes/CityscapesResNet18/resnet18_SFSegNets.pth with
strict=True, which proves that the trees match the checkpoints; both files are in torch's legacy format, which
torch.load only reads with weights_only=False, so that is what it is given here (files of the reference checkout),
with map_location='cpu'.

Files:
  image_resnet18_families_keys.npz   the keys and shapes (no values) of both checkpoints and of the other file of the
                                     Cityscapes directory (resnet18.pth, not loadable), and the state-dict keys of the
                                     reference wrapper of every class;
  image_resnet18_families_<family>_layer0.npz   the checkpoint's real layer0 parameters and buffers under the
                                     wrapper's keys (conv.0.*), and an eval-mode and a train-mode TruncatedLayer0 step
                                     on them (input and upstream gradient from the hash generator, checksums stored);
  image_resnet18_families_<case>.npz  seeded cases (CASES), recorded as the ADE20K cases of
                                     oracle/make_golden_image_resnet18.py are, plus num_batches_tracked after the step.
tests/test_image_resnet18_families_oracle.py checks oracle/image_resnet18_families_oracle.py against every fixture."""
import contextlib
import functools
import os

import numpy as np
import torch

from oracle import image_resnet18_oracle as R
from oracle.make_golden_image_resnet18 import case_inputs, case_upstream, load_reference_image

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
LAYERS = ["Layer0", "Layer1", "Layer2", "Layer3", "Layer4"]
CLASSES = ([f"ResNet18Truncated{n}" for n in LAYERS[:4]] + ["ResNet18TruncatedLayer4"] + [f"ResNet18{n}" for n in LAYERS]
           + ["ResNet18Pyramid"] + [f"CityscapesResNet18Truncated{n}" for n in LAYERS]
           + [f"CityscapesResNet18{n}" for n in LAYERS] + ["CityscapesResNet18Pyramid", "CityscapesResNet18"])
CKPT = {"imagenet": ("imagenet", "resnet18", "resnet18.pth"),
        "cityscapes": ("cityscapes", "CityscapesResNet18", "resnet18_SFSegNets.pth"),
        "other": ("cityscapes", "CityscapesResNet18", "resnet18.pth")}
LAYER0 = {"imagenet": ("ResNet18TruncatedLayer0", (2, 3, 50, 66), 21),
          "cityscapes": ("CityscapesResNet18TruncatedLayer0", (2, 3, 52, 66), 22)}


@contextlib.contextmanager
def legacy_load():
    """torch.load with weights_only=False and map_location='cpu' while the reference reads its own checkpoints (legacy
    format; the Cityscapes one was saved from CUDA)."""
    load = torch.load
    torch.load = functools.partial(load, weights_only=False, map_location="cpu")
    try:
        yield
    finally:
        torch.load = load


def checkpoint_path(image, which):
    return os.path.join(image.PRETRAINED_DIR, *CKPT[which])


def make_keys(image):
    out = {}
    for which in CKPT:
        sd = torch.load(checkpoint_path(image, which), map_location="cpu", weights_only=False)
        out[f"{which}:keys"] = np.array(list(sd))
        out[f"{which}:shapes"] = np.array([str(tuple(v.shape)) for v in sd.values()])
    with legacy_load():
        for cls in CLASSES:
            out[f"keys:{cls}"] = np.array(list(getattr(image, cls)().state_dict()))
    return out


def step(net, x, gy, out, prefix=""):
    """One forward and backward of net in float64; y, the norms, the running stats and counters after the step."""
    x = x.clone().requires_grad_(True)
    y = net(x)
    if gy is None:
        gy = case_upstream(tuple(y.shape), int(out["seed"]))
    g = torch.autograd.grad(y, [x] + list(net.parameters()), gy)
    out[f"{prefix}y"] = y.detach().float().numpy()
    out[f"{prefix}y_norm"] = np.float64(y.detach().norm())
    out[f"{prefix}gx"] = g[0].float().numpy()
    out[f"{prefix}gx_norm"] = np.float64(g[0].norm())
    for tag, ((k, _), gp) in enumerate(zip(net.named_parameters(), g[1:])):
        out[f"{prefix}gnorm:{k}"] = np.float64(gp.norm())
        out[f"{prefix}gproj:{k}"] = np.float64((gp * R.projection(int(out["seed"]), tag, tuple(gp.shape))).sum())
    for k, v in net.state_dict().items():
        if k.endswith((".running_mean", ".running_var", ".num_batches_tracked")):
            out[f"{prefix}after:{k}"] = v.numpy()


def make_layer0(image, family):
    """The real layer0 slice, and an eval-mode and a train-mode TruncatedLayer0 step on it in float64."""
    cls, shape, seed = LAYER0[family]
    with legacy_load():
        ref = getattr(image, cls)()
    out = {k: v.numpy() for k, v in ref.state_dict().items()}
    out["seed"] = np.int64(seed)
    _, x = case_inputs(ref, shape, seed)
    out["checksum:x"] = np.float64(x.sum())
    for mode in ("eval", "train"):
        with legacy_load():
            net = getattr(image, cls)().double().train(mode == "train")
        step(net, x, None, out, f"{mode}:")
    return out


# name -> (class, kwargs, training, input shape, seed): the 7x7 stem at odd sides, every BasicBlock layer with its
# downsample, an eval step, the unpadded pool dropping a row and a column, the Cityscapes 128 -> 64 downsample at
# stride 1, the whole CityscapesResNet18 and both Pyramids
CASES = {
    "rn_tl4_train": ("ResNet18TruncatedLayer4", {}, True, (2, 3, 61, 45), 11),
    "rn_layer2_eval": ("ResNet18Layer2", {}, False, (1, 64, 15, 18), 12),
    "rn_pyramid_train": ("ResNet18Pyramid", {"scale_factor": -1}, True, (2, 3, 8, 10), 13),
    "cs_tl4_train": ("CityscapesResNet18TruncatedLayer4", {}, True, (2, 3, 60, 44), 14),
    "cs_layer1_train": ("CityscapesResNet18Layer1", {}, True, (2, 128, 9, 11), 15),
    "cs_full_train": ("CityscapesResNet18", {}, True, (2, 3, 50, 66), 16),
    "cs_pyramid_eval": ("CityscapesResNet18Pyramid", {}, False, (2, 3, 10, 8), 17),
}


def make_case(image, cls, kwargs, training, shape, seed):
    net = getattr(image, cls)(pretrained=False, **kwargs).double().train(training)
    state, x = case_inputs(net, shape, seed)
    net.load_state_dict(state, strict=True)
    out = {"seed": np.int64(seed)}
    step(net, x, None, out)
    for k, v in state.items():
        if k.endswith((".weight", ".bias", ".running_mean", ".running_var")):
            out[f"checksum:{k}"] = np.float64(v.double().sum())
    out["checksum:x"] = np.float64(x.sum())
    return out


def main():
    os.environ.setdefault("PYTORCH_JIT", "0")
    image = load_reference_image()
    files = [("keys", make_keys(image))] + [(f"{f}_layer0", make_layer0(image, f)) for f in LAYER0]
    files += [(name, make_case(image, *spec)) for name, spec in CASES.items()]
    for name, d in files:
        path = os.path.join(OUT, f"image_resnet18_families_{name}.npz")
        np.savez_compressed(path, **d)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
