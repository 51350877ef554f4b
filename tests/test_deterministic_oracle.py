"""The ordered oracle of the deterministic backwards (oracle/deterministic_oracle.py) against a plain
Python loop over float32 scalars and against autograd through the reference-path oracle, plus the
host-side argument checks of the deterministic C entry points (no launch).  Runs without a GPU."""
import ctypes

import numpy as np
import pytest
import torch

from deepviewagg_b200 import _lib
from oracle import deterministic_oracle as D
from oracle import pooling_oracle as O

f32 = np.float32


def _bilin_scalar(px, py, H, W, map_w, map_h):
    """Scalar float32 restatement of the bilinear footprint: ((row, col) x 4, weight x 4), clamped."""
    cy, cx = f32(py) / f32(map_h - 1), f32(px) / f32(map_w - 1)
    p0, p1 = cy * f32(H) + f32(0.5), cx * f32(W) + f32(0.5)
    top, bottom = np.floor(p0), np.floor(p0 + f32(1))
    left, right = np.floor(p1), np.floor(p1 + f32(1))
    wts = [abs((p0 - bottom) * (p1 - right)), abs((p0 - bottom) * (p1 - left)),
           abs((p0 - top) * (p1 - right)), abs((p0 - top) * (p1 - left))]
    r = [min(max(int(top) - 1, 0), H - 1), min(max(int(bottom) - 1, 0), H - 1)]
    c = [min(max(int(left) - 1, 0), W - 1), min(max(int(right) - 1, 0), W - 1)]
    return [(r[0], c[0]), (r[0], c[1]), (r[1], c[0]), (r[1], c[1])], [f32(w) for w in wts]


def _loop_grad(x, g, images, pixels, aptr, reduce, mapping_size=None):
    """The contract written as nested loops: first arg from the forward values, then every element
    accumulated contribution by contribution in ascending (p, k)."""
    B, C, H, W = x.shape
    out = np.zeros((B, H, W, C), dtype=f32)
    for w in range(len(aptr) - 1):
        p0, p1 = int(aptr[w]), int(aptr[w + 1])
        n = p1 - p0
        b = min(max(int(images[w]), 0), B - 1)
        foot = []
        for p in range(p0, p1):
            px, py = int(pixels[p, 0]), int(pixels[p, 1])
            if mapping_size is None:
                foot.append(([(min(max(py, 0), H - 1), min(max(px, 0), W - 1))], [None]))
            else:
                foot.append(_bilin_scalar(px, py, H, W, *mapping_size))
        for c in range(C):
            best = None
            if reduce in ("max", "min") and n >= 2:
                vals = []
                for corners, wts in foot:
                    if mapping_size is None:
                        vals.append(f32(x[b, c, corners[0][0], corners[0][1]]))
                    else:
                        v = f32(0)
                        for k, ((r, cc), wk) in enumerate(zip(corners, wts)):
                            t = f32(wk * f32(x[b, c, r, cc]))
                            v = t if k == 0 else f32(v + t)
                        vals.append(v)
                best = 0
                for i in range(1, n):
                    if (vals[i] > vals[best]) if reduce == "max" else (vals[i] < vals[best]):
                        best = i
            for i, (corners, wts) in enumerate(foot):
                if best is not None and i != best:
                    continue
                val = f32(g[w, c])
                if reduce == "mean":
                    val = f32(val / f32(n))
                for (r, cc), wk in zip(corners, wts):
                    v = val if wk is None else f32(wk * val)
                    out[b, r, cc, c] = f32(out[b, r, cc, c] + v)
    return out


def _case(seed, B, C, H, W, Vw, map_size=None, oob=False):
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, 4, Vw)
    counts[: Vw // 5] = 0                                          # empty views
    counts[Vw // 5: 2 * Vw // 5] = 1
    aptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    P = int(aptr[-1])
    mw, mh = map_size if map_size else (W, H)
    pix = np.stack([rng.integers(0, mw, P), rng.integers(0, mh, P)], 1).astype(np.int64)
    pix[1::3] = pix[0:-1:3][: len(pix[1::3])]                       # duplicated pixels (inside and across views)
    if map_size:
        pix[::7, 0] = mw - 1                                          # corners clamped at the border
        pix[::11, 1] = mh - 1
        pix[::13] = 0
    if oob:
        pix[::9, 0] = W + 3                                           # clamped like the forward
        pix[::10, 1] = -2
    images = rng.integers(0, B, Vw).astype(np.int64)
    x = rng.standard_normal((B, C, H, W)).astype(f32)
    x[x < -0.5] = 0                                                   # ties for max / min
    g = rng.standard_normal((Vw, C)).astype(f32)
    return x, g, images, pix, aptr


def _ordered(x, g, images, pix, aptr, reduce, mapping_size=None):
    B, C, H, W = x.shape
    arg = None
    if reduce in ("max", "min"):
        arg = D.first_arg(D.gathered_values(x, images, pix, aptr, mapping_size), aptr, reduce)
    return D.map_grad_ordered((B, H, W, C), g, images, pix, aptr, reduce, arg, mapping_size)


@pytest.mark.parametrize("reduce", ["sum", "mean", "max", "min"])
@pytest.mark.parametrize("interp", [False, True])
def test_ordered_oracle_equals_scalar_loop(reduce, interp):
    for seed in range(3):
        msz = (29, 17) if interp else None
        x, g, images, pix, aptr = _case(seed, 2, 3, 6, 7, 30, map_size=msz, oob=not interp)
        got = _ordered(x, g, images, pix, aptr, reduce, msz)
        want = _loop_grad(x, g, images, pix, aptr, reduce, msz)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (reduce, interp, seed)


def test_ordered_oracle_reuse_heavy_buckets():
    """4x the map resolution: every map pixel collects many bilinear contributions."""
    x, g, images, pix, aptr = _case(5, 1, 2, 3, 4, 60, map_size=(16, 12))
    for reduce in ("sum", "max"):
        got = _ordered(x, g, images, pix, aptr, reduce, (16, 12))
        want = _loop_grad(x, g, images, pix, aptr, reduce, (16, 12))
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), reduce


@pytest.mark.parametrize("reduce", ["sum", "mean", "max", "min"])
def test_ordered_oracle_matches_autograd(reduce):
    gen = torch.Generator().manual_seed(3)
    B, C, H, W, Vw = 3, 8, 9, 11, 200
    counts = torch.randint(0, 4, (Vw,), generator=gen)
    aptr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)])
    P = int(aptr[-1])
    img = torch.randint(0, B, (Vw,), generator=gen)
    pix = torch.stack([torch.randint(0, W, (P,), generator=gen), torch.randint(0, H, (P,), generator=gen)], 1)
    fmap = torch.randn(B, C, H, W, generator=gen)
    w = torch.randn(Vw, C, generator=gen)
    fo = fmap.clone().requires_grad_(True)
    ref = O.segment_csr(O.feature_map_gather(fo, img, pix, aptr), aptr, reduce=reduce)
    rg = torch.autograd.grad((ref * w).sum(), fo)[0].permute(0, 2, 3, 1).numpy()
    got = _ordered(fmap.numpy(), w.numpy(), img.numpy(), pix.numpy(), aptr.numpy(), reduce)
    assert np.abs(got - rg).max() <= 1e-6 * max(1.0, float(np.abs(rg).max()))


@pytest.mark.parametrize("tag", ["half", "quarter"])
def test_bilinear_footprint_reproduces_interpolation_oracle(tag):
    """Interpolating with the ordered oracle's bilinear footprint gives, bit for bit, the values of
    oracle/image_oracle.py and of the reference's sparse_interpolation (tests/golden fixture)."""
    from conftest import load_golden
    from oracle.image_oracle import sparse_interpolation_pixels
    g = load_golden("sparse_interpolation")
    W, H, _ = [int(v) for v in g[f"{tag}_size"]]
    x, pix, batch = g[f"{tag}_x"].numpy(), g[f"{tag}_pix"].numpy(), g[f"{tag}_batch"].numpy()
    B, C, h, w = x.shape
    (top, bottom, left, right), (w_tl, w_tr, w_bl, w_br) = D.bilinear_footprint(pix, (W, H), h, w)
    padded = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)), mode="edge")
    b = batch.astype(np.int64)

    def at(r, c):
        return padded[b, :, r.astype(np.int64), c.astype(np.int64)]

    out = w_tl[:, None] * at(top, left) + w_tr[:, None] * at(top, right)
    out = (out + w_bl[:, None] * at(bottom, left)) + w_br[:, None] * at(bottom, right)
    want = sparse_interpolation_pixels(x, pix, batch, (W, H))
    assert np.array_equal(out.astype(f32).view(np.uint32), want.view(np.uint32))
    assert np.array_equal(want, g[f"{tag}_out"].numpy())


def test_rows_ordered_oracle():
    rng = np.random.default_rng(1)
    V, R, C = 300, 40, 5
    src = rng.standard_normal((V, C)).astype(f32)
    idx = rng.integers(-2, R + 2, V)
    want = np.zeros((R, C), dtype=f32)
    for v in range(V):
        if 0 <= idx[v] < R:
            for c in range(C):
                want[idx[v], c] = f32(want[idx[v], c] + src[v, c])
    got = D.scatter_add_rows_ordered(src, idx, R)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_det_entry_points_validate_arguments():
    """Bad sizes, null pointers and short workspaces are refused before anything is launched."""
    lib = _lib.load()
    E = _lib.DVA_EINVAL
    fake = ctypes.c_void_p(256)             # never dereferenced: every call below fails validation
    for name in ("dva_gather_pool_bwd_det_workspace_bytes", "dva_interp_pool_bwd_det_workspace_bytes"):
        fn = getattr(lib, name)
        assert fn(2, 8, 8, 100) > fn(2, 8, 8, 10) > 0
        assert fn(-1, 8, 8, 10) == 0
    assert lib.dva_interp_pool_bwd_det_workspace_bytes(2, 8, 8, 100) > lib.dva_gather_pool_bwd_det_workspace_bytes(2, 8, 8, 100)
    ws = lib.dva_gather_pool_bwd_det_workspace_bytes(2, 8, 8, 10)
    gp = lib.dva_gather_pool_bwd_det
    # (grad_out, cl, img, pix, i16, aptr, arg, gfmap, B, C, H, W, Vw, P, reduce, dtype, ws, ws_bytes, stream)
    assert gp(fake, 1, fake, fake, 0, fake, None, fake, -1, 4, 8, 8, 5, 10, 0, 0, fake, ws, None) == E
    assert gp(fake, 1, fake, fake, 0, fake, None, None, 2, 4, 8, 8, 5, 10, 0, 0, fake, ws, None) == E
    assert gp(None, 1, fake, fake, 0, fake, None, fake, 2, 4, 8, 8, 5, 10, 0, 0, fake, ws, None) == E
    assert gp(fake, 1, fake, fake, 0, fake, None, fake, 2, 4, 8, 8, 5, 10, 0, 0, None, ws, None) == E
    assert gp(fake, 1, fake, fake, 0, fake, None, fake, 2, 4, 8, 8, 5, 10, 0, 0, fake, ws - 1, None) == E
    assert b"workspace too small" in lib.dva_last_error()
    assert gp(fake, 1, fake, fake, 0, fake, None, fake, 2, 4, 8, 8, 5, 10, 2, 0, fake, ws, None) == E   # max: no arg
    assert gp(fake, 1, fake, fake, 0, fake, None, fake, 2, 4, 8, 8, 5, 10, 7, 0, fake, ws, None) == E   # reduce
    assert gp(fake, 1, fake, fake, 0, fake, None, fake, 2, 4, 8, 8, 5, 10, 0, 9, fake, ws, None) == E   # dtype
    assert gp(fake, 1, fake, fake, 0, fake, None, fake, 0, 4, 8, 8, 5, 10, 0, 0, fake, ws, None) == E   # empty map
    assert b"gather_pool_bwd_det" in lib.dva_last_error()
    wsi = lib.dva_interp_pool_bwd_det_workspace_bytes(2, 8, 8, 10)
    ip = lib.dva_interp_pool_bwd_det
    assert ip(fake, 1, fake, fake, 0, fake, None, fake, 2, 4, 8, 8, 1, 16, 5, 10, 0, 0, fake, wsi, None) == E   # map_w < 2
    assert ip(fake, 1, fake, fake, 0, fake, None, fake, 2, 4, 8, 8, 16, 16, 5, 10, 0, 0, fake, ws, None) == E   # ws
    assert b"interp_pool_bwd_det" in lib.dva_last_error()
    wr = lib.dva_scatter_add_rows_det_workspace_bytes(100, 10)
    assert wr > 0 and lib.dva_scatter_add_rows_det_workspace_bytes(-1, 10) == 0
    sr = lib.dva_scatter_add_rows_det
    assert sr(fake, fake, fake, -1, 10, 4, 0, fake, wr, None) == E
    assert sr(fake, fake, None, 100, 10, 4, 0, fake, wr, None) == E
    assert sr(fake, None, fake, 100, 10, 4, 0, fake, wr, None) == E
    assert sr(fake, fake, fake, 100, 10, 4, 0, None, wr, None) == E
    assert sr(fake, fake, fake, 100, 10, 4, 0, fake, wr - 1, None) == E
    assert sr(fake, fake, fake, 100, 10, 4, 5, fake, wr, None) == E
    assert b"scatter_add_rows_det" in lib.dva_last_error()
