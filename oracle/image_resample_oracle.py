"""Pillow's 8-bit resize restated in numpy (oracle; test infrastructure).

PIL.Image.resize(size, box=box) with the default BICUBIC filter on an RGB image runs ImagingResample:
per axis, precompute_coeffs gives every output index a window [xmin, xmin + xmax) of source indices and
float64 weights bicubic((x + xmin - center + 0.5) / filterscale) normalised by their sequential sum;
normalize_coeffs_8bpc turns them into int32 weights scaled by 2^22 (rounded half away from zero).  A
horizontal pass over the source rows the vertical pass needs writes a uint8 temporary (clipped), then a
vertical pass writes the output; an axis that does not change is skipped.  Every sum starts at 2^21 and is
shifted right by 22 and clamped to [0, 255].

Written per output index with Python floats (IEEE double, one rounding per operation), so it shares no code
with the vectorised tables of deepviewagg_b200.ops.
"""
import math

import numpy as np

PRECISION_BITS = 32 - 8 - 2


def bicubic(x, a=-0.5):
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coefficients(in_size, in0, in1, out_size):
    """-> (bounds [out, 2] (xmin, count), int32 weights [out, ksize])"""
    in0, in1 = np.float32(in0), np.float32(in1)
    scale = float(np.float32(in1 - in0)) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    bounds = np.zeros((out_size, 2), dtype=np.int64)
    kk = np.zeros((out_size, ksize), dtype=np.int64)
    for xx in range(out_size):
        center = float(in0) + (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        for x, v in enumerate(w):
            kk[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def _clip8(s):
    return np.clip(s >> PRECISION_BITS, 0, 255).astype(np.uint8)


def _pass(img, bounds, kk, axis):
    """convolution of an [H, W, C] uint8 image along axis 1 (horizontal) or 0 (vertical)"""
    src = img.astype(np.int64)
    n_out = bounds.shape[0]
    shape = list(img.shape)
    shape[axis] = n_out
    out = np.empty(shape, dtype=np.uint8)
    for o in range(n_out):
        xmin, cnt = bounds[o]
        win = np.take(src, np.arange(xmin, xmin + cnt), axis=axis)
        w = kk[o, :cnt].reshape((-1, 1, 1) if axis == 0 else (1, -1, 1))
        s = (1 << (PRECISION_BITS - 1)) + (win * w).sum(axis=axis)
        if axis == 0:
            out[o] = _clip8(s)
        else:
            out[:, o] = _clip8(s)
    return out


def resize(img, size, box=None):
    """img [H, W, C] uint8, size (W_out, H_out), box (x0, y0, x1, y1) or None -> [H_out, W_out, C] uint8,
    PIL.Image.fromarray(img).resize(size, box=box) byte for byte."""
    H, W = img.shape[:2]
    Wo, Ho = size
    box = (0, 0, W, H) if box is None else tuple(box)
    box = tuple(float(np.float32(b)) for b in box)
    need_h = Wo != W or box[0] != 0 or box[2] != Wo
    need_v = Ho != H or box[1] != 0 or box[3] != Ho
    xb, xk = coefficients(W, box[0], box[2], Wo)
    yb, yk = coefficients(H, box[1], box[3], Ho)
    out = img
    if need_h:
        first, last = yb[0, 0], yb[-1, 0] + yb[-1, 1]
        out = _pass(img[first:last], xb, xk, axis=1)
        yb = yb.copy()
        yb[:, 0] -= first
    if need_v:
        out = _pass(out, yb, yk, axis=0)
    return out.copy()
