"""Ordered CPU reference of the deterministic backwards (TEST INFRASTRUCTURE ONLY -- see
oracle/__init__.py; never imported by the product path).

Under torch.use_deterministic_algorithms(True) the feature-map gradient of ops.gather_pool /
ops.interp_pool / ops.sparse_interpolation_pixels and the rows scatter-add of ops.view_attention /
ops.heuristic_pool are summed in a fixed order (DESIGN.md section 4.3).  This module accumulates the
same contributions in the same order with float32 numpy arithmetic, so the GPU result must equal it
bit for bit:
  contributions (p, k) of map element (b, y, x, c): pixel slot p of view w in atomic-CSR order, k = 0
    (plain gather) or k = 0..3 = corners tl, tr, bl, br (bilinear), ascending (p, k);
  value: g = float32(grad_out[w, c]); mean: g / n_w; max / min: only when n_w == 1 or the slot is the
    first arg-max / arg-min of the view for channel c; bilinear: w_k * value;
  sum: from +0.0 with one float32 addition per contribution (np.add.at, unbuffered, in index order).
"""
import numpy as np

from oracle.image_oracle import sparse_interpolation_pixels


def bilinear_footprint(pix, mapping_size, h, w):
    """Corners and weights of the bilinear sample of every pixel, in float32 and in the order of
    oracle/image_oracle.py's sparse_interpolation_pixels (the reference's image.py:1280-1281, 143-162);
    tests/test_deterministic_oracle.py checks that interpolating with this footprint reproduces that
    function bit for bit on the reference fixture.  pix [P,2] integer (x, y) at the mapping resolution
    `mapping_size` = (W, H) of a [h, w] map.  Returns (top, bottom, left, right) as float32 row / column
    indices in the 1-px replicate-padded frame and the weights (w_tl, w_tr, w_bl, w_br) float32 [P]."""
    f32 = np.float32
    W, H = mapping_size
    px = np.asarray(pix)[:, 0].astype(f32)
    py = np.asarray(pix)[:, 1].astype(f32)
    p0 = (py / f32(H - 1)) * f32(h) + f32(0.5)
    p1 = (px / f32(W - 1)) * f32(w) + f32(0.5)
    top, bottom = np.floor(p0), np.floor(p0 + f32(1))
    left, right = np.floor(p1), np.floor(p1 + f32(1))
    w_tl = np.abs((p0 - bottom) * (p1 - right))
    w_tr = np.abs((p0 - bottom) * (p1 - left))
    w_bl = np.abs((p0 - top) * (p1 - right))
    w_br = np.abs((p0 - top) * (p1 - left))
    return (top, bottom, left, right), (w_tl, w_tr, w_bl, w_br)


def _slots(atomic_ptr):
    aptr = np.asarray(atomic_ptr).astype(np.int64)
    counts = aptr[1:] - aptr[:-1]
    view = np.repeat(np.arange(counts.size, dtype=np.int64), counts)     # view of slots aptr[0] .. aptr[-1]
    return aptr, counts, view


def first_arg(vals, atomic_ptr, reduce):
    """[Vw, C] int64: absolute slot of the first arg-max (max) / arg-min (min) of every view and
    channel (the forward's choice), -1 for empty views."""
    aptr, counts, view = _slots(atomic_ptr)
    vals = np.asarray(vals, dtype=np.float32)[aptr[0]:aptr[-1]]
    Vw, C = counts.size, vals.shape[1]
    arg = np.full((Vw, C), -1, dtype=np.int64)
    nz = counts > 0
    if not nz.any():
        return arg
    starts = (aptr[:-1] - aptr[0])[nz]
    ext = (np.maximum if reduce == "max" else np.minimum).reduceat(vals, starts, axis=0)
    full = np.zeros((Vw, C), dtype=np.float32)
    full[nz] = ext
    slot = np.arange(aptr[0], aptr[-1], dtype=np.int64)[:, None].repeat(C, 1)
    big = np.iinfo(np.int64).max
    cand = np.where(vals == full[view], slot, big)
    arg[nz] = np.minimum.reduceat(cand, starts, axis=0)
    return arg


def gathered_values(x_nchw, images, pixels, atomic_ptr, mapping_size=None):
    """[P, C] float32 values the forward pools: the (clamped) map pixel, or its bilinear sample."""
    x = np.asarray(x_nchw, dtype=np.float32)
    B, C, h, w = x.shape
    aptr, counts, view = _slots(atomic_ptr)
    pix = np.asarray(pixels).astype(np.int64)
    b = np.clip(np.asarray(images).astype(np.int64)[view], 0, B - 1)
    pix = pix[aptr[0]:aptr[-1]]
    if mapping_size is None:
        return x[b, :, np.clip(pix[:, 1], 0, h - 1), np.clip(pix[:, 0], 0, w - 1)]
    return sparse_interpolation_pixels(x, pix, b, mapping_size)


def map_grad_ordered(shape_bhwc, grad_out, images, pixels, atomic_ptr, reduce, arg=None, mapping_size=None):
    """Map gradient [B, H, W, C] float32 (channels-last) of gather_pool / interp_pool in the
    deterministic order.  arg: first_arg(...) of the forward values, needed for max / min."""
    B, H, W, C = shape_bhwc
    f32 = np.float32
    aptr, counts, view = _slots(atomic_ptr)
    g = np.asarray(grad_out, dtype=np.float32)
    pix = np.asarray(pixels).astype(np.int64)[aptr[0]:aptr[-1]]
    slot = np.arange(aptr[0], aptr[-1], dtype=np.int64)
    n = counts[view]
    val = g[view]                                                       # [S, C]
    if reduce == "mean":
        val = val / n.astype(f32)[:, None]
    if reduce in ("max", "min"):
        on = (n[:, None] == 1) | (np.asarray(arg)[view] == slot[:, None])
        val = np.where(on, val, f32(0))      # adding +0.0 leaves the sum (never -0.0) unchanged
    b = np.clip(np.asarray(images).astype(np.int64)[view], 0, B - 1)
    if mapping_size is None:
        key = (b * H + np.clip(pix[:, 1], 0, H - 1)) * W + np.clip(pix[:, 0], 0, W - 1)
        keys, vals = key, val
    else:
        (top, bottom, left, right), weights = bilinear_footprint(pix, mapping_size, H, W)
        rows = [np.clip(r.astype(np.int64) - 1, 0, H - 1) for r in (top, bottom)]
        cols = [np.clip(c.astype(np.int64) - 1, 0, W - 1) for c in (left, right)]
        corner = [(rows[0], cols[0]), (rows[0], cols[1]), (rows[1], cols[0]), (rows[1], cols[1])]
        keys = np.stack([(b * H + r) * W + c for r, c in corner], 1).reshape(-1)          # ascending (p, k)
        vals = np.stack([wk[:, None] * val for wk in weights], 1).reshape(-1, C)
    out = np.zeros((B * H * W, C), dtype=np.float32)
    np.add.at(out, keys, vals.astype(np.float32))
    return out.reshape(B, H, W, C)


def scatter_add_rows_ordered(src, idx, n_rows):
    """dst [n_rows, C] float32: row r = sum over ascending v with idx[v] == r of float32(src[v]),
    from +0.0; indices outside [0, n_rows) are skipped."""
    src = np.asarray(src, dtype=np.float32)
    idx = np.asarray(idx).astype(np.int64)
    out = np.zeros((n_rows, src.shape[1]), dtype=np.float32)
    ok = (idx >= 0) & (idx < n_rows)
    np.add.at(out, idx[ok], src[ok])
    return out
