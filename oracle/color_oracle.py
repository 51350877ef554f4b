"""float32 numpy restatement of torchvision's tensor colour arithmetic, as the reference's ColorJitter,
ToFloatImage and Normalize run it (core/data_transform/multimodal/image.py:1221-1283, torchvision
transforms/_functional_tensor.py: rgb_to_grayscale, _blend, adjust_brightness / contrast / saturation,
normalize; transforms.ColorJitter.get_params).

Every float32 operation is a separate numpy ufunc call (no FMA, no reassociation): Python scalars are rounded
to float32 before they multiply a tensor, `1 - ratio` is taken in float64 first, sums run left to right, and
uint8 conversion truncates.  The contrast mean is an argument, so the oracle runs with torch's fp32
`torch.mean` (the reference) or with the exact mean (this package)."""
import numpy as np
import torch

F32 = np.float32
OPS = ("brightness", "contrast", "saturation")


def check_input(v):
    """torchvision's ColorJitter._check_input for a scalar: [max(0, 1 - v), 1 + v], None when v == 0."""
    if v < 0:
        raise ValueError("a ColorJitter factor must be non negative")
    lo, hi = max(1.0 - float(v), 0.0), 1.0 + float(v)
    return None if lo == hi == 1.0 else (lo, hi)


def draw(brightness, contrast, saturation):
    """torchvision's ColorJitter.get_params on the CPU default generator, hue off: (fn_idx [4] int64, b, c, s)."""
    fn_idx = torch.randperm(4)
    out = [fn_idx]
    for rng in (brightness, contrast, saturation):
        out.append(None if rng is None else float(torch.empty(1).uniform_(rng[0], rng[1])))
    return tuple(out)


def grayscale(x):
    """[..., 3, H, W] uint8 -> [..., H, W] uint8: (0.2989 r + 0.587 g) + 0.114 b in fp32, truncated"""
    f = x.astype(F32)
    r, g, b = f[..., 0, :, :], f[..., 1, :, :], f[..., 2, :, :]
    return ((F32(0.2989) * r + F32(0.587) * g) + F32(0.114) * b).astype(np.uint8)


def blend(img1, other, ratio):
    """_blend: fp32(ratio) * img1 + fp32(1 - ratio) * other, clamped to [0, 255], truncated to uint8"""
    v = F32(ratio) * img1.astype(F32) + F32(1.0 - float(ratio)) * other
    return np.clip(v, F32(0), F32(255)).astype(np.uint8)


def exact_mean(gray):
    """float32(float64(S) / float64(H W)) per image of [B, H, W] uint8, S the integer sum"""
    s = gray.reshape(gray.shape[0], -1).astype(np.int64).sum(axis=1)
    return (s.astype(np.float64) / float(gray.shape[-1] * gray.shape[-2])).astype(F32)


def torch_mean(gray):
    """the reference's mean: torch.mean of the fp32 grayscale over (C, H, W), per image"""
    t = torch.from_numpy(np.ascontiguousarray(gray)).unsqueeze(1).float()
    return torch.mean(t, dim=(-3, -2, -1)).numpy().astype(F32)


def apply_op(x, op, ratio, mean=None):
    """one adjust_* on [B, 3, H, W] uint8; for contrast, `mean` [B] fp32 (None: the exact mean)"""
    if op == "brightness":
        return blend(x, np.zeros_like(x, dtype=F32), ratio)
    if op == "saturation":
        return blend(x, grayscale(x)[:, None].astype(F32), ratio)
    if op == "contrast":
        m = exact_mean(grayscale(x)) if mean is None else np.asarray(mean, dtype=F32)
        return blend(x, m.reshape(-1, 1, 1, 1), ratio)
    raise ValueError(op)


def color_jitter(x, fn_idx, factors, means=None):
    """ColorJitter.forward on [B, 3, H, W] uint8 with drawn fn_idx and factors (b, c, s; None = off).  `means`:
    the contrast mean [B] to use (None: the exact one).  Returns (out, [(mean used, image before
    the contrast op)]) -- one item when contrast is on, to flag near-integer blends."""
    steps = []
    for fn in [int(i) for i in fn_idx]:
        if fn > 2 or factors[fn] is None:
            continue
        op = OPS[fn]
        if op == "contrast":
            g = grayscale(x)
            m = exact_mean(g) if means is None else np.asarray(means, dtype=F32)
            steps.append((m, x.copy()))
            x = apply_op(x, op, factors[fn], m)
        else:
            x = apply_op(x, op, factors[fn])
    return x, steps


def contrast_near_integer(x_before, ratio, mean_a, mean_b):
    """[B, 3, H, W] bool: pixels whose contrast blend value truncates differently under mean_a and mean_b"""
    a = F32(ratio) * x_before.astype(F32)
    q = F32(1.0 - float(ratio))
    va = np.clip(a + q * np.asarray(mean_a, F32).reshape(-1, 1, 1, 1), F32(0), F32(255)).astype(np.uint8)
    vb = np.clip(a + q * np.asarray(mean_b, F32).reshape(-1, 1, 1, 1), F32(0), F32(255)).astype(np.uint8)
    return va != vb


def to_float(x):
    """ToFloatImage: x.float() / 255 with true division"""
    return x.astype(F32) / F32(255)


def normalize(x, mean, std):
    """torchvision normalize: (x - mean_c) / std_c in fp32, [C, 1, 1] fp32 statistics"""
    m = np.asarray(mean, dtype=F32).reshape(-1, 1, 1)
    s = np.asarray(std, dtype=F32).reshape(-1, 1, 1)
    return (x.astype(F32) - m) / s


def color_input(kind, B, H, W):
    """[B, 3, H, W] uint8 inputs of the colour fixtures, from a closed formula (stored as shape and sum only):
      'formula'  (7 i + 50 c + 3 y + 5 w + (y w mod 11)) mod 256
      'edges'    image 0 all 0, image 1 all 255, then 'formula'
      'ramps'    image 0 a grey ramp along w, image 1 bands of the 8 saturated colours ({0, 255}^3), then
                 per-channel ramps with different slopes along w and y"""
    i, c, y, w = np.meshgrid(np.arange(B), np.arange(3), np.arange(H), np.arange(W), indexing="ij")
    x = (7 * i + 50 * c + 3 * y + 5 * w + (y * w) % 11) % 256
    if kind == "edges":
        x = np.where(i == 0, 0, np.where(i == 1, 255, x))
    elif kind == "ramps":
        grey = (w * 255) // max(W - 1, 1)
        band = (w * 8) // W
        sat = ((band >> c) & 1) * 255
        slopes = (y * (c + 1) * 255 // max(H - 1, 1) + w * (3 - c) * 2) % 256
        x = np.where(i == 0, grey, np.where(i == 1, sat, slopes))
    elif kind != "formula":
        raise ValueError(kind)
    return x.astype(np.uint8)
