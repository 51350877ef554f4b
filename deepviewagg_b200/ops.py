"""Autograd operators over the C ABI (include/dva_b200.h).

Each function mirrors one operator of the reference's multimodal path (same argument meaning,
same empty-segment / tie / eps semantics) and is backed ONLY by the sm_90a kernels of
libdva_b200.so: CPU tensors or a missing library raise.  Reference citations are relative to the
reference repository root.
"""
import contextlib
import math
import os

import numpy as np
import torch

# torch.amp integration (SURVEY 8b "Autograd / AMP / recompute"): every autograd.Function's forward is
# wrapped in torch.amp.custom_fwd and its backward in custom_bwd, so that (a) the backward runs under
# the autocast state of its forward and (b) the tensor-core projection is computed from fp32 operands
# (cast_inputs) whatever dtype autocast hands it -- never less precise than the reference's fp16
# autocast path (models/segmentation/sparseconv3d.py:24).  The feature operators (segment / gather /
# attention) run in the dtype of their inputs (fp32, bf16 or fp16 storage, fp32 accumulation), which
# is what torch_scatter does under autocast.
_fwd = torch.amp.custom_fwd(device_type="cuda")
_fwd_f32 = torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
_bwd = torch.amp.custom_bwd(device_type="cuda")

from . import _lib
from ._lib import DTYPE_CODES, REDUCE_CODES, dtype_code, launch, require_cuda


def _as_2d(src):
    if src.dim() == 1:
        return src.contiguous().view(-1, 1)
    if src.dim() == 2:
        return src.contiguous()
    return src.contiguous().view(src.shape[0], -1)


def _check_csr(csr_idx, device):
    if csr_idx.dtype != torch.int64:
        raise TypeError("csr_idx must be a LongTensor (core/multimodal/csr.py:54)")
    if csr_idx.dim() != 1 or csr_idx.numel() < 1:
        raise ValueError("csr_idx must be a 1D pointer tensor of size n_groups + 1")
    if csr_idx.device != device:
        raise RuntimeError("csr_idx must live on the device of the features")
    return csr_idx.contiguous()


# --------------------------------------------------------------------------------------------
# segment_csr  (torch_scatter.segment_csr as used at pooling.py:63,289,295,519,525,628,787,807)
# --------------------------------------------------------------------------------------------
class _SegmentCSR(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, src, csr_idx, reduce):
        require_cuda(src, csr_idx)
        code = REDUCE_CODES[reduce]
        shape = src.shape
        s2 = _as_2d(src)
        csr_idx = _check_csr(csr_idx, src.device)
        n_seg, n_items, K = csr_idx.numel() - 1, s2.shape[0], s2.shape[1]
        # outputs are allocated in their final shape: returning a view from a custom Function
        # would forbid the in-place updates the reference applies downstream (Gating,
        # pooling.py:705-711)
        out = torch.empty((n_seg,) + tuple(shape[1:]), dtype=src.dtype, device=src.device)
        arg = None
        if code in (2, 3):
            arg = torch.empty((n_seg, K), dtype=torch.int64, device=src.device)
        launch("dva_segment_csr_fwd", src.device, s2, csr_idx, out, arg, n_seg, n_items, K, code, dtype_code(s2))
        ctx.code, ctx.n_items, ctx.in_shape = code, n_items, shape
        ctx.save_for_backward(csr_idx, arg)
        return out

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        csr_idx, arg = ctx.saved_tensors
        g2 = _as_2d(grad_out)
        n_seg, K = g2.shape
        gsrc = torch.empty(ctx.in_shape, dtype=g2.dtype, device=g2.device)
        launch("dva_segment_csr_bwd", g2.device, g2, csr_idx, arg, gsrc, n_seg, ctx.n_items, K, ctx.code,
               dtype_code(g2))
        return gsrc, None, None


def segment_csr(src, indptr, out=None, reduce="sum"):
    """torch_scatter.segment_csr(src, indptr, out=None, reduce) along dim 0.

    Empty segments reduce to 0 for every mode (pooling.py:870); max/min route the gradient to
    the first arg-max/min row of the segment.
    """
    if out is not None:
        raise NotImplementedError("segment_csr(out=...) is not used by the reference path")
    if reduce not in REDUCE_CODES:
        raise ValueError(f"unknown reduce '{reduce}'")
    return _SegmentCSR.apply(src, indptr, reduce)


def segment_csr_arg(src, indptr, reduce="max"):
    """(values, first-arg rows) like torch_scatter.segment_max_csr; arg = n_items when empty."""
    require_cuda(src, indptr)
    s2 = _as_2d(src)
    indptr = _check_csr(indptr, src.device)
    n_seg, n_items, K = indptr.numel() - 1, s2.shape[0], s2.shape[1]
    out = torch.empty((n_seg, K), dtype=src.dtype, device=src.device)
    arg = torch.empty((n_seg, K), dtype=torch.int64, device=src.device)
    launch("dva_segment_csr_fwd", src.device, s2, indptr, out, arg, n_seg, n_items, K, REDUCE_CODES[reduce],
           dtype_code(s2))
    tail = tuple(src.shape[1:])
    return out.view((n_seg,) + tail), arg.view((n_seg,) + tail)


# --------------------------------------------------------------------------------------------
# gather_csr (pooling.py:813-841)
# --------------------------------------------------------------------------------------------
class _GatherCSR(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, src, csr_idx, n_items):
        require_cuda(src, csr_idx)
        s2 = _as_2d(src)
        csr_idx = _check_csr(csr_idx, src.device)
        n_seg, K = csr_idx.numel() - 1, s2.shape[1]
        out = torch.empty((n_items,) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
        launch("dva_gather_csr", src.device, s2, csr_idx, out, n_seg, n_items, K, dtype_code(s2))
        ctx.in_shape = src.shape
        ctx.save_for_backward(csr_idx)
        return out

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        (csr_idx,) = ctx.saved_tensors
        g2 = _as_2d(grad_out)
        n_items, K = g2.shape
        n_seg = csr_idx.numel() - 1
        gsrc = torch.empty(ctx.in_shape, dtype=g2.dtype, device=g2.device)
        launch("dva_segment_csr_fwd", g2.device, g2, csr_idx, gsrc, None, n_seg, n_items, K, REDUCE_CODES["sum"],
               dtype_code(g2))
        return gsrc, None, None


def gather_csr(src, csr_idx, n_items=None):
    """Redistribute segment-level rows to their items (pooling.py:813-841).

    `n_items` avoids the device->host read of csr_idx[-1] when the caller knows V already.
    """
    if not torch.is_floating_point(src):
        raise ValueError("`gather_csr` can only be computed over tensors with floating point data types.")
    if csr_idx.dim() != 1:
        raise ValueError("`gather_csr` can only be computed over 1D CSR indices.")
    if src.dim() > 2:
        raise NotImplementedError("`gather_csr` can only be computed over 1D or 2D source tensors.")
    if n_items is None:
        n_items = int(csr_idx[-1].item())
    return _GatherCSR.apply(src, csr_idx, n_items)


def segment_gather_csr(src, csr_idx, reduce="sum"):
    """segment_csr then gather_csr (pooling.py:844-856)."""
    return gather_csr(segment_csr(src, csr_idx, reduce=reduce), csr_idx, n_items=src.shape[0])


# --------------------------------------------------------------------------------------------
# segment_softmax_csr (pooling.py:758-810)
# --------------------------------------------------------------------------------------------
class _SegmentSoftmaxCSR(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, src, csr_idx, eps, scaling):
        require_cuda(src, csr_idx)
        s2 = _as_2d(src)
        csr_idx = _check_csr(csr_idx, src.device)
        n_seg, n_items, K = csr_idx.numel() - 1, s2.shape[0], s2.shape[1]
        out = torch.empty(src.shape, dtype=src.dtype, device=src.device)
        launch("dva_segment_softmax_csr_fwd", src.device, s2, csr_idx, out, n_seg, n_items, K, float(eps),
               int(bool(scaling)), dtype_code(s2))
        ctx.scaling, ctx.in_shape = bool(scaling), src.shape
        ctx.save_for_backward(csr_idx, out)
        return out

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        csr_idx, out = ctx.saved_tensors
        g2 = _as_2d(grad_out)
        n_items, K = g2.shape
        gsrc = torch.empty(ctx.in_shape, dtype=g2.dtype, device=g2.device)
        launch("dva_segment_softmax_csr_bwd", g2.device, out, g2, csr_idx, gsrc, csr_idx.numel() - 1, n_items, K,
               int(ctx.scaling), dtype_code(g2))
        return gsrc, None, None, None


def segment_softmax_csr(src, csr_idx, eps=1e-12, scaling=False):
    """Equivalent of scatter_softmax for CSR indices (pooling.py:758-810), same signature."""
    if not torch.is_floating_point(src):
        raise ValueError("`segment_csr_softmax` can only be computed over tensors with floating point data types.")
    if csr_idx.dim() != 1:
        raise ValueError("`segment_csr_softmax` can only be computed over 1D CSR indices.")
    if src.dim() > 2:
        raise NotImplementedError("`segment_csr_softmax` can only be computed over 1D or 2D source tensors.")
    return _SegmentSoftmaxCSR.apply(src, csr_idx, eps, scaling)


# --------------------------------------------------------------------------------------------
# fused view attention (modules.py:518 + pooling.py:285-300 / 515-530)
# --------------------------------------------------------------------------------------------
def _scatter_add_rows(src, idx, n_rows):
    """fp32 [n_rows, C] with dst[idx[v]] += src[v] (dva_scatter_add_rows).  Under
    torch.use_deterministic_algorithms(True): dva_scatter_add_rows_det (every row summed in ascending v)."""
    src = src.contiguous()
    V, C = src.shape
    if torch.are_deterministic_algorithms_enabled():
        dst = torch.empty((n_rows, C), dtype=torch.float32, device=src.device)
        ws = _lib.workspace(_lib.load().dva_scatter_add_rows_det_workspace_bytes(V, n_rows), src.device)
        launch("dva_scatter_add_rows_det", src.device, src, idx.contiguous(), dst, V, n_rows, C, dtype_code(src),
               ws, ws.numel())
        return dst
    dst = torch.zeros((n_rows, C), dtype=torch.float32, device=src.device)
    launch("dva_scatter_add_rows", src.device, src, idx.contiguous(), dst, V, n_rows, C, dtype_code(src))
    return dst


def fused_groups_supported(num_groups):
    return 1 <= num_groups <= 32 and (num_groups & (num_groups - 1)) == 0


class _ViewAttention(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, x, idx, compat, csr_idx, gate_w, gate_b, num_groups, group_scaling, eps,
                idx_is_permutation):
        require_cuda(x, idx, compat, csr_idx, gate_w, gate_b)
        x = x.contiguous()
        compat = compat.float().contiguous()
        csr_idx = _check_csr(csr_idx, x.device)
        N, V, G = csr_idx.numel() - 1, compat.shape[0], int(num_groups)
        R, C = x.shape
        if compat.shape[1] != G:
            raise ValueError(f"compatibilities must be [V,{G}], got {tuple(compat.shape)}")
        idx64 = 0
        if idx is not None:
            if idx.dtype not in (torch.int32, torch.int64):
                raise TypeError("idx must be int32 or int64")
            idx = idx.contiguous()
            idx64 = int(idx.dtype == torch.int64)
            if idx.numel() != V:
                raise ValueError("idx must hold one row id per view")
        elif R != V:
            raise ValueError("x must hold one row per view when idx is None")
        gw = gate_w.detach().float().contiguous().view(-1) if gate_w is not None else None
        gb = gate_b.detach().float().contiguous().view(-1) if gate_b is not None else None
        out = torch.empty((N, C), dtype=x.dtype, device=x.device)
        att = torch.empty((V, G), dtype=torch.float32, device=x.device)
        seg_max = torch.empty((N, G), dtype=torch.float32, device=x.device)
        seg_den = torch.empty((N, G), dtype=torch.float32, device=x.device)
        seg_arg = torch.empty((N, G), dtype=torch.int32, device=x.device)
        launch("dva_view_attention_fwd", x.device, x, idx, idx64, compat, csr_idx, gw, gb, out, att, seg_max,
               seg_den, seg_arg, N, V, R, C, G, int(bool(group_scaling)), float(eps), dtype_code(x))
        ctx.cfg = (N, V, R, C, G, bool(group_scaling), idx64, bool(idx_is_permutation),
                   gate_w.shape if gate_w is not None else None,
                   gate_b.shape if gate_b is not None else None,
                   gate_w.dtype if gate_w is not None else None)
        ctx.save_for_backward(x, idx, compat, csr_idx, gw, gb, seg_max, seg_den, seg_arg)
        ctx.mark_non_differentiable(att, seg_max)
        return out, att, seg_max

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out, _ga, _gm):
        x, idx, compat, csr_idx, gw, gb, seg_max, seg_den, seg_arg = ctx.saved_tensors
        N, V, R, C, G, scaling, idx64, is_perm, w_shape, b_shape, w_dtype = ctx.cfg
        grad_out = grad_out.contiguous()
        scatter = int(idx is not None and is_perm and R == V)
        gx_rows = torch.empty((V, C), dtype=x.dtype, device=x.device)
        gcompat = torch.empty((V, G), dtype=torch.float32, device=x.device)
        ggate, ws = None, None                      # the workspace holds the gate-gradient partials only
        if gw is not None:
            ggate = torch.empty((2, G), dtype=torch.float32, device=x.device)
            ws = _lib.workspace(_lib.load().dva_view_attention_bwd_workspace_bytes(G), x.device)
        launch("dva_view_attention_bwd", x.device, x, idx, idx64, compat, csr_idx, gw, gb, grad_out, seg_max,
               seg_den, seg_arg, gx_rows, gcompat, ggate, scatter, N, V, R, C, G, int(scaling), dtype_code(x), ws,
               0 if ws is None else ws.numel())
        if idx is None or scatter:
            gx = gx_rows
        else:  # general (non-injective) gather: accumulate duplicated rows (red.global.add.v4.f32 kernel)
            gx = _scatter_add_rows(gx_rows, idx.long(), R).to(x.dtype)
        g_w = ggate[0].view(w_shape).to(w_dtype) if gw is not None else None
        g_b = ggate[1].view(b_shape).to(w_dtype) if gw is not None else None
        return gx, None, gcompat, None, g_w, g_b, None, None, None, None


def view_attention(x, compat, csr_idx, num_groups, idx=None, gate_weight=None, gate_bias=None,
                   group_scaling=False, eps=1e-12, idx_is_permutation=False):
    """Fused gather + group softmax + weighted sum (+ gating).

    Returns (x_pool [N,C], attentions [V,G], seg_max [N,G]) where
      attentions = segment_softmax_csr(compat, csr_idx, scaling=group_scaling)
      x_pool     = segment_csr(x[idx] * expand_group_feat(attentions), csr_idx, 'sum')
                   * expand_group_feat(tanh(relu(w * segment_csr(compat,'max') + b)))   if gating
    i.e. the chain modules.py:518 -> pooling.py:285-300. `idx` (int32/int64 [V], optional) is the
    row of `x` feeding each view (e.g. ImageData.view_cat_sorting, image.py:1549-1574).
    """
    if not fused_groups_supported(num_groups):
        raise NotImplementedError("fused view attention needs num_groups to be a power of two <= 32")
    if (gate_weight is None) != (gate_bias is None):
        raise ValueError("gate_weight and gate_bias go together")
    return _ViewAttention.apply(x, idx, compat, csr_idx, gate_weight, gate_bias, num_groups,
                                group_scaling, eps, idx_is_permutation)


# --------------------------------------------------------------------------------------------
# ragged Q.K compatibilities (pooling.py:499-512)
# --------------------------------------------------------------------------------------------
class _QKScores(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, keys, queries, csr_idx, num_groups, scale):
        require_cuda(keys, queries, csr_idx)
        k32, q32 = keys.float().contiguous(), queries.float().contiguous()
        csr_idx = _check_csr(csr_idx, keys.device)
        N, V, G = csr_idx.numel() - 1, k32.shape[0], int(num_groups)
        D = k32.shape[1] // G
        if k32.shape[1] != G * D or q32.shape != (N, G * D):
            raise ValueError("keys must be [V,G*D] and queries [N,G*D]")
        compat = torch.empty((V, G), dtype=torch.float32, device=keys.device)
        launch("dva_qk_scores_fwd", keys.device, k32, q32, csr_idx, compat, N, V, G, D, float(scale))
        ctx.cfg = (N, V, G, D, float(scale), keys.dtype, queries.dtype)
        ctx.save_for_backward(k32, q32, csr_idx)
        return compat

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, gcompat):
        k32, q32, csr_idx = ctx.saved_tensors
        N, V, G, D, scale, kd, qd = ctx.cfg
        gcompat = gcompat.float().contiguous()
        gk, gq = torch.empty_like(k32), torch.empty_like(q32)
        launch("dva_qk_scores_bwd", k32.device, k32, q32, csr_idx, gcompat, gk, gq, N, V, G, D, scale)
        return gk.to(kd), gq.to(qd), None, None, None


def qk_scores(keys, queries, csr_idx, num_groups, dim_scaling=True):
    """compat[v,g] = sum_d K[v,g,d] Q[point(v),g,d] (/ sqrt(D) if dim_scaling), pooling.py:499-512."""
    D = keys.shape[1] // num_groups
    scale = 1.0 / math.sqrt(D) if dim_scaling else 1.0
    return _QKScores.apply(keys, queries, csr_idx, num_groups, scale)


# --------------------------------------------------------------------------------------------
# heuristic pool (pooling.py:129-152)
# --------------------------------------------------------------------------------------------
class _HeuristicPool(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, x_mod, x_map, csr_idx, feat, use_max):
        require_cuda(x_mod, x_map, csr_idx)
        x_mod = x_mod.contiguous()
        m32 = x_map.float().contiguous()
        csr_idx = _check_csr(csr_idx, x_mod.device)
        N, V, C = csr_idx.numel() - 1, x_mod.shape[0], x_mod.shape[1]
        out = torch.empty((N, C), dtype=x_mod.dtype, device=x_mod.device)
        arg = torch.empty((N,), dtype=torch.int64, device=x_mod.device)
        launch("dva_heuristic_pool_fwd", x_mod.device, x_mod, m32, m32.shape[1], int(feat), csr_idx, out, arg, N,
               V, C, int(bool(use_max)), dtype_code(x_mod))
        ctx.V = V
        ctx.save_for_backward(arg)
        return out

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        (arg,) = ctx.saved_tensors
        # each point picks a distinct view (arg == V: none, skipped by the kernel)
        g = _scatter_add_rows(grad_out.contiguous(), arg, ctx.V).to(grad_out.dtype)
        return g, None, None, None, None


def heuristic_pool(x_mod, x_map, csr_idx, feat, mode="max"):
    return _HeuristicPool.apply(x_mod, x_map, csr_idx, feat, mode == "max")


# --------------------------------------------------------------------------------------------
# fused feature-map gather + atomic pool (image.py:1285 + pooling.py:63)
# --------------------------------------------------------------------------------------------
def _transpose_last2(t, B, R, S):
    """[B,R,S] -> [B,S,R] copy through dva_transpose_last2 (t contiguous)."""
    out = torch.empty_like(t)
    launch("dva_transpose_last2", t.device, t, out, B, R, S, dtype_code(t))
    return out


# NCHW maps: when at least this share of the map's pixels is gathered, one transposition to
# channels-last (2 x map bytes) beats reading every element through its own 32-byte sector
_NCHW_TRANSPOSE_SHARE = 0.25


_INDEX_CHECKS = {"on": os.environ.get("DVA_CHECK_INDICES", "0") not in ("", "0")}


def set_index_checks(on):
    """Validate pixel / image indices of every gather_pool / interp_pool call on the host (one
    device->host read per call) and raise IndexError like the reference's
    `x[feature_map_indexing]` (image.py:1285).  Off by default: the kernels clamp out-of-range
    indices into the map (memory-safe, no synchronisation).  Also switched on by DVA_CHECK_INDICES=1."""
    _INDEX_CHECKS["on"] = bool(on)


def _validate_gather_indices(images, pixels, B, W, H):
    if pixels.numel() == 0:
        return
    lo = torch.stack([pixels[:, 0].min(), pixels[:, 1].min(), images.min()]).tolist()
    hi = torch.stack([pixels[:, 0].max(), pixels[:, 1].max(), images.max()]).tolist()
    if lo[0] < 0 or lo[1] < 0 or lo[2] < 0 or hi[0] >= W or hi[1] >= H or hi[2] >= B:
        raise IndexError(f"mapping out of bounds for feature maps [B={B}, H={H}, W={W}]: pixels x in "
                         f"[{lo[0]}, {hi[0]}], y in [{lo[1]}, {hi[1]}], image ids in [{lo[2]}, {hi[2]}] "
                         f"(stale or mis-scaled mapping?)")


class _GatherPool(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, fmap, images, pixels, atomic_ptr, reduce, channels_last, mapping_size):
        require_cuda(fmap, images, pixels, atomic_ptr)
        fmap = fmap.contiguous()
        via_cl = False
        if channels_last:
            B, H, W, C = fmap.shape
        else:
            B, C, H, W = fmap.shape
            n_corner = 1 if mapping_size is None else 4
            if (fmap.dtype in DTYPE_CODES and C % (16 // fmap.element_size()) == 0 and B <= 65535
                    and pixels.shape[0] * n_corner >= _NCHW_TRANSPOSE_SHARE * B * H * W):
                # the reference's layout (image.py:1884): transpose once, then the channels-last kernels
                fmap = _transpose_last2(fmap, B, C, H * W).view(B, H, W, C)
                channels_last, via_cl = True, True
        images = images.long().contiguous()
        if pixels.dtype not in (torch.int16, torch.int32):
            pixels = pixels.int()
        pixels = pixels.contiguous()
        atomic_ptr = _check_csr(atomic_ptr, fmap.device)
        Vw, P, code = atomic_ptr.numel() - 1, pixels.shape[0], REDUCE_CODES[reduce]
        if images.numel() != Vw:
            raise ValueError("images must hold one image id per view (atomic_ptr.numel() - 1)")
        if _INDEX_CHECKS["on"]:
            lim = (W, H) if mapping_size is None else mapping_size
            _validate_gather_indices(images, pixels.long(), B, int(lim[0]), int(lim[1]))
        out = torch.empty((Vw, C), dtype=fmap.dtype, device=fmap.device)
        arg = torch.empty((Vw, C), dtype=torch.int64, device=fmap.device) if code in (2, 3) else None
        head = (fmap, int(channels_last), images, pixels, int(pixels.dtype == torch.int16), atomic_ptr, out, arg,
                B, C, H, W)
        tail = (Vw, P, code, dtype_code(fmap))
        if mapping_size is None:
            launch("dva_gather_pool_fwd", fmap.device, *head, *tail)
        else:
            launch("dva_interp_pool_fwd", fmap.device, *head, int(mapping_size[0]), int(mapping_size[1]), *tail)
        ctx.cfg = (B, C, H, W, Vw, P, code, bool(channels_last), fmap.shape, fmap.dtype, mapping_size, via_cl)
        ctx.save_for_backward(images, pixels, atomic_ptr, arg)
        return out

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        images, pixels, atomic_ptr, arg = ctx.saved_tensors
        B, C, H, W, Vw, P, code, cl, shape, dt, mapping_size, via_cl = ctx.cfg
        grad_out = grad_out.contiguous()
        dev = grad_out.device
        # torch.use_deterministic_algorithms(True): the map gradient is reduced per map pixel in a fixed
        # order (the _det entry points write every element) instead of accumulated with fp32 atomics
        det = torch.are_deterministic_algorithms_enabled()
        gf = (torch.empty if det else torch.zeros)(shape, dtype=torch.float32, device=dev)
        head = (grad_out, int(cl), images, pixels, int(pixels.dtype == torch.int16), atomic_ptr, arg, gf, B, C, H, W)
        tail = (Vw, P, code, dtype_code(grad_out))
        msz = () if mapping_size is None else (int(mapping_size[0]), int(mapping_size[1]))
        name = "dva_gather_pool_bwd" if mapping_size is None else "dva_interp_pool_bwd"
        if det:
            ws = _lib.workspace(getattr(_lib.load(), name + "_det_workspace_bytes")(B, H, W, P), dev)
            launch(name + "_det", dev, *head, *msz, *tail, ws, ws.numel())
        else:
            launch(name, dev, *head, *msz, *tail)
        if via_cl:      # gradient of the NCHW input: transpose the channels-last map gradient back
            gf = _transpose_last2(gf, B, H * W, C).view(B, C, H, W)
        return gf.to(dt), None, None, None, None, None, None


def gather_pool(fmap, images, pixels, atomic_ptr, reduce="max", channels_last=False):
    """segment_csr(fmap[(images_per_pixel, :, py, px)], atomic_ptr, reduce) without the [P,C] copy."""
    return _GatherPool.apply(fmap, images, pixels, atomic_ptr, reduce, channels_last, None)


def interp_pool(fmap, images, pixels, atomic_ptr, mapping_size, reduce="max", channels_last=False):
    """segment_csr(sparse_interpolation(fmap, pixels / (mapping_size - 1), images_per_pixel),
    atomic_ptr, reduce) (image.py:1278-1283 + pooling.py:63) in one kernel.  `pixels` are (x, y)
    at the mapping resolution `mapping_size` = (W_map, H_map); padding mode 'border'."""
    return _GatherPool.apply(fmap, images, pixels, atomic_ptr, reduce, channels_last,
                             (int(mapping_size[0]), int(mapping_size[1])))


def sparse_interpolation_pixels(fmap, images_per_pixel, pixels, mapping_size, channels_last=False):
    """Per-pixel bilinear features [P, C] (image.py:1278-1283): the pooled kernel with one pixel per
    segment."""
    P = pixels.shape[0]
    aptr = torch.arange(P + 1, dtype=torch.int64, device=fmap.device)
    return _GatherPool.apply(fmap, images_per_pixel, pixels, aptr, "sum", channels_last,
                             (int(mapping_size[0]), int(mapping_size[1])))


# --------------------------------------------------------------------------------------------
# fused BatchNorm1d + LeakyReLU over [rows, C] (base_modules.py:38-48, 131-156)
# --------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _fp32_running(running_mean, running_var):
    """The running buffers as the contiguous fp32 arrays the training kernels update IN PLACE through raw
    pointers.  A buffer of another dtype or layout (e.g. a module converted with .half()) is staged through an
    fp32 copy, which is written back when the block ends."""
    bufs = (running_mean, running_var)
    staged = tuple(b if b is None or (b.dtype == torch.float32 and b.is_contiguous()) else b.float().contiguous()
                   for b in bufs)
    yield staged
    for buf, tmp in zip(bufs, staged):
        if tmp is not buf:
            buf.copy_(tmp)


def _bn_apply(z, gamma, beta, mean, invstd, eps, slope):
    """act(gamma (z - mean) invstd + beta) on given statistics: dva_bn_act_fwd with training = 0, which reads
    only mean / invstd (also passed for the running buffers it requires) and no workspace."""
    y = torch.empty_like(z)
    launch("dva_bn_act_fwd", z.device, z, gamma, beta, mean, mean, mean, invstd, y, z.shape[0], z.shape[1],
           float(eps), 0.0, float(slope), 0, dtype_code(z), None, 0)
    return y


class _BNAct(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, z, weight, bias, running_mean, running_var, training, momentum, eps, slope,
                pre_mean=None, pre_invstd=None):
        require_cuda(z, weight, bias, running_mean, running_var)
        z = z.contiguous()
        R, C = z.shape
        dev = z.device
        gamma = weight.detach().float().contiguous() if weight is not None else None
        beta = bias.detach().float().contiguous() if bias is not None else None
        if training and pre_mean is None:
            mean = torch.empty(C, dtype=torch.float32, device=dev)
            invstd = torch.empty(C, dtype=torch.float32, device=dev)
            y = torch.empty_like(z)
            ws = _lib.workspace(_lib.load().dva_bn_workspace_bytes(R, C), dev)
            with _fp32_running(running_mean, running_var) as (rm, rv):
                launch("dva_bn_act_fwd", dev, z, gamma, beta, rm, rv, mean, invstd, y, R, C, float(eps),
                       float(momentum), float(slope), 1, dtype_code(z), ws, ws.numel())
        else:
            if training:
                # batch statistics already taken in the producing GEMM's epilogue (ops.linear_bn_act): apply only;
                # the backward still differentiates through the batch statistics (ctx keeps training = True)
                mean, invstd = pre_mean, pre_invstd
            else:
                for name, buf in (("running_mean", running_mean), ("running_var", running_var)):
                    if buf.dtype != torch.float32 or not buf.is_contiguous():
                        raise TypeError(f"{name} must be a contiguous float32 buffer in eval mode")
                mean = running_mean.float().contiguous()
                invstd = torch.rsqrt(running_var.float() + eps).contiguous()
            y = _bn_apply(z, gamma, beta, mean, invstd, eps, slope)
        ctx.cfg = (R, C, float(slope), bool(training), weight is not None, bias is not None,
                   weight.dtype if weight is not None else None)
        ctx.save_for_backward(z, gamma, beta, mean, invstd)
        return y

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        z, gamma, beta, mean, invstd = ctx.saved_tensors
        R, C, slope, training, has_w, has_b, wdt = ctx.cfg
        dy = dy.contiguous()
        dz = torch.empty_like(z)
        sums = torch.empty((2, C), dtype=torch.float32, device=z.device)
        ws = _lib.workspace(_lib.load().dva_bn_workspace_bytes(R, C), z.device)
        launch("dva_bn_act_bwd", z.device, dy, z, gamma, beta, mean, invstd, dz, sums, R, C, slope, int(training),
               dtype_code(z), ws, ws.numel())
        gw = sums[1].to(wdt) if has_w else None
        gb = sums[0].to(wdt) if has_b else None
        return dz, gw, gb, None, None, None, None, None, None, None, None


def _uses_batch_stats(bn):
    """nn.BatchNorm1d normalises with the batch statistics in training and when it keeps no running ones."""
    return bn.training or (bn.running_mean is None and bn.running_var is None)


def _bn_step(bn):
    """nn.BatchNorm1d's bookkeeping for one forward: num_batches_tracked += 1 in training; returns the running
    buffers to update (None when not tracked) and the momentum (1 / num_batches_tracked, a cumulative average,
    when bn.momentum is None)."""
    momentum = 0.0 if bn.momentum is None else bn.momentum
    if bn.training and bn.track_running_stats and bn.num_batches_tracked is not None:
        bn.num_batches_tracked.add_(1)
        if bn.momentum is None:
            momentum = 1.0 / float(bn.num_batches_tracked)
    rm = bn.running_mean if bn.track_running_stats else None
    rv = bn.running_var if bn.track_running_stats else None
    return rm, rv, momentum


def batch_norm_act(z, bn, negative_slope=1.0):
    """act(BatchNorm1d(z)) for z [rows, C] with the statistics / running-average semantics of
    nn.BatchNorm1d (training: batch statistics over all rows, momentum update of the running
    buffers, num_batches_tracked += 1).  `bn` is the nn.BatchNorm1d holding the parameters;
    negative_slope = 1 gives plain BatchNorm, 0.2 the MLP layers of the pools."""
    rm, rv, momentum = _bn_step(bn)
    return _BNAct.apply(z, bn.weight, bn.bias, rm, rv, _uses_batch_stats(bn), momentum, bn.eps, negative_slope)


# --------------------------------------------------------------------------------------------
# dense projection of the MLP layers on wgmma tensor cores (base_modules.py:42)
# --------------------------------------------------------------------------------------------
_GEMM_PRECISION = {"mode": 0}


def set_gemm_precision(mode):
    """Kept for API stability: 'fp32' or 'tf32'.  Every projection kernel is 3xTF32 (fp32-grade
    accuracy) since round 2, so both modes run the same code."""
    _GEMM_PRECISION["mode"] = {"fp32": 0, "tf32": 1}[mode]


def _aligned16(t):
    """t, or a copy of it when its data does not start on a 16-byte boundary (e.g. a contiguous view at an odd
    storage offset): the wgmma, bnstats and fused-layer kernels read their rows with TMA / 16-byte loads."""
    return t if t is None or t.data_ptr() % 16 == 0 else t.clone()


def _tc_gemm(a, b, layout, n_out):
    """layout 0: D[M,n_out] = a[M,K] . b[n_out,K]^T;  1: D[M,n_out] = a[M,K] . b[K,n_out];
    2: D[N,n_out] = a[M,N]^T . b[M,n_out]  -- through dva_linear_gemm."""
    prec = _GEMM_PRECISION["mode"]
    if layout == 2:
        M, N = a.shape
        K = n_out
        out = torch.empty((N, K), dtype=torch.float32, device=a.device)
    else:
        M, K = a.shape
        N = n_out
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    lib = _lib.load()
    if (a.data_ptr() | b.data_ptr()) % 16 and not lib.dva_linear_gemm_skinny(M, N, K, layout):
        a, b = _aligned16(a), _aligned16(b)                    # the skinny kernels take any alignment
    ws = _lib.workspace(lib.dva_linear_gemm_workspace_bytes(M, N, K, layout, prec), a.device)
    launch("dva_linear_gemm", a.device, a, b, out, M, N, K, layout, prec, ws, ws.numel())
    return out


def _linear_grads(ctx, gz):
    """(dX, dW) of z = x @ w.T, each only when its input needs it, from the (x, w) the forward saved."""
    x, w = ctx.saved_tensors
    gz = gz.float().contiguous()
    gx = _tc_gemm(gz, w, 1, w.shape[1]) if ctx.needs_input_grad[0] else None
    # dW = dZ^T X: [out,in] result reduced over all rows -- stream-K split over the SMs
    gw = _tc_gemm(gz, x, 2, x.shape[1]) if ctx.needs_input_grad[1] else None
    return gx, gw


def _linear_bnstats(x, w, running_mean, running_var, momentum, eps):
    """z = x @ w.T (fp32, contiguous) with the batch statistics of z's columns taken in the GEMM epilogue
    (dva_linear_bnstats_fwd), which also updates the running buffers: returns (z, mean, invstd)."""
    M, K = x.shape
    N = w.shape[0]
    x, w = _aligned16(x), _aligned16(w)
    z = torch.empty((M, N), dtype=torch.float32, device=x.device)
    mean = torch.empty(N, dtype=torch.float32, device=x.device)
    invstd = torch.empty(N, dtype=torch.float32, device=x.device)
    ws = _lib.workspace(_lib.load().dva_linear_bnstats_workspace_bytes(N, K), x.device)
    with _fp32_running(running_mean, running_var) as (rm, rv):
        launch("dva_linear_bnstats_fwd", x.device, x, w, z, M, N, K, float(eps), float(momentum), mean, invstd, rm,
               rv, ws, ws.numel())
    return z, mean, invstd


def tc_gemm_supported(x, weight):
    """True for 2-D CUDA floating-point inputs with at least one row: every such projection runs on
    this library's kernels (K, N <= 64: skinny kernels, any K / N; otherwise the wgmma kernels, whose
    16-byte TMA rows need K and N to be multiples of 4 -- other widths are zero-padded by `linear`)."""
    return bool(x.is_cuda and weight.is_cuda and x.dim() == 2 and x.shape[0] > 0
                and x.is_floating_point() and weight.is_floating_point())


class _Linear(torch.autograd.Function):
    @staticmethod
    @_fwd_f32
    def forward(ctx, x, weight):
        require_cuda(x, weight)
        x, w = x.float().contiguous(), weight.float().contiguous()
        ctx.save_for_backward(x, w)
        ctx.dtypes = (x.dtype, weight.dtype)
        return _tc_gemm(x, w, 0, w.shape[0])

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, gz):
        return _linear_grads(ctx, gz)


class _LinearStats(torch.autograd.Function):
    """z = x @ weight.T with the BatchNorm batch statistics of z's columns taken in the GEMM epilogue
    (dva_linear_bnstats_fwd): returns (z, mean, invstd); running buffers are updated in place."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, x, weight, running_mean, running_var, momentum, eps):
        require_cuda(x, weight)
        # aligned before saving, so that the backward's wgmma dW reads the same copy
        x, w = _aligned16(x.float().contiguous()), _aligned16(weight.float().contiguous())
        z, mean, invstd = _linear_bnstats(x, w, running_mean, running_var, momentum, eps)
        ctx.save_for_backward(x, w)
        ctx.mark_non_differentiable(mean, invstd)
        return z, mean, invstd

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, gz, _gm, _gi):
        return (*_linear_grads(ctx, gz), None, None, None, None)


class _MLPLayer(torch.autograd.Function):
    """One narrow MLP layer act(BatchNorm1d(x @ weight.T)) in training mode (base_modules.py:38-48) as ONE autograd
    node: forward = GEMM with the batch statistics in its epilogue (dva_linear_bnstats_fwd) + the apply pass;
    backward = the statistics pass + ONE kernel for dz (kept on chip), dX and dW (dva_mlp_layer_bwd)."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, momentum, eps, slope):
        require_cuda(x, weight, gamma, beta)
        # aligned before saving: dva_mlp_layer_bwd reads the saved x with 16-byte loads too
        x, w = _aligned16(x.float().contiguous()), _aligned16(weight.float().contiguous())
        g = gamma.detach().float().contiguous() if gamma is not None else None
        b = beta.detach().float().contiguous() if beta is not None else None
        z, mean, invstd = _linear_bnstats(x, w, running_mean, running_var, momentum, eps)
        y = _bn_apply(z, g, b, mean, invstd, eps, slope)
        ctx.cfg = (float(slope), gamma is not None, beta is not None,
                   gamma.dtype if gamma is not None else (beta.dtype if beta is not None else None), weight.dtype)
        ctx.save_for_backward(x, w, z, g, b, mean, invstd)
        return y

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        x, w, z, g, b, mean, invstd = ctx.saved_tensors
        slope, has_g, has_b, pdt, wdt = ctx.cfg
        M, K = x.shape
        N = w.shape[0]
        dy = _aligned16(dy.float().contiguous())
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = torch.empty_like(w)
        sums = torch.empty((2, N), dtype=torch.float32, device=x.device)
        ws = _lib.workspace(_lib.load().dva_mlp_layer_bwd_workspace_bytes(M, N, K), x.device)
        launch("dva_mlp_layer_bwd", x.device, dy, z, x, w, g, b, mean, invstd, dx, dw, sums, M, N, K, slope, ws,
               ws.numel())
        gw = sums[1].to(pdt) if has_g else None
        gb = sums[0].to(pdt) if has_b else None
        return dx, (dw.to(wdt) if ctx.needs_input_grad[1] else None), gw, gb, None, None, None, None, None


# The fused backward (3xTF32 on mma.sync) replaces three kernels with one pass; at K = 64 it needs 2 CTAs per SM of
# registers / shared memory and the unfused chain (dX on the wgmma kernel) is used -> layers with K <= 32 only.
# This cut-off was chosen on another GPU and is not re-measured on the H100 (tools/bench_layer.py measures it).
_MLP_LAYER_FUSED = {"on": os.environ.get("DVA_MLP_LAYER_FUSED", "1") != "0", "max_k": 32}


def linear_bn_act(x, weight, bn, negative_slope=1.0):
    """act(BatchNorm1d(x @ weight.T)): one MLP layer of the pools (base_modules.py:38-48).  In training,
    when the layer is wide enough for the wgmma kernel and has at most 128 output channels, the batch
    statistics come out of the GEMM epilogue (2 passes over the activations instead of 3); otherwise
    linear() followed by batch_norm_act()."""
    lib = _lib.load()
    M, K = x.shape
    N = weight.shape[0]
    if not (_uses_batch_stats(bn) and x.is_cuda and M > 0 and K % 4 == 0
            and lib.dva_linear_bnstats_supported(M, N, K)):
        return batch_norm_act(linear(x, weight), bn, negative_slope=negative_slope)
    rm, rv, momentum = _bn_step(bn)
    if (_MLP_LAYER_FUSED["on"] and K <= _MLP_LAYER_FUSED["max_k"] and lib.dva_mlp_layer_bwd_supported(M, N, K)
            and torch.is_grad_enabled()
            and (x.requires_grad or weight.requires_grad)):
        return _MLPLayer.apply(x, weight, bn.weight, bn.bias, rm, rv, momentum, bn.eps, negative_slope)
    z, mean, invstd = _LinearStats.apply(x, weight, rm, rv, momentum, bn.eps)
    return _BNAct.apply(z, bn.weight, bn.bias, rm, rv, True, momentum, bn.eps, negative_slope, mean, invstd)


def linear(x, weight):
    """x @ weight.T for a bias-free nn.Linear weight [out, in] (base_modules.py:42), always on this
    library's kernels, computed from fp32 operands (also under autocast).  Wide layers whose K or N is
    not a multiple of 4 are zero-padded to the next multiple (exact: the padding contributes 0)."""
    if not tc_gemm_supported(x, weight):
        raise RuntimeError("ops.linear needs 2-D CUDA floating-point operands with at least one row "
                           "(no CPU / library fallback)")
    out_dtype = x.dtype if not torch.is_autocast_enabled("cuda") else torch.float32
    K, N = x.shape[1], weight.shape[0]
    if not (K <= 64 and N <= 64):
        pk, pn = (-K) % 4, (-N) % 4
        if pk:
            x = torch.nn.functional.pad(x, (0, pk))
            weight = torch.nn.functional.pad(weight, (0, pk))
        if pn:
            weight = torch.nn.functional.pad(weight, (0, 0, 0, pn))
        z = _Linear.apply(x, weight)
        z = z[:, :N] if pn else z
    else:
        z = _Linear.apply(x, weight)
    return z if z.dtype == out_dtype or out_dtype not in (torch.float16, torch.bfloat16) else z.to(out_dtype)


# --------------------------------------------------------------------------------------------
# image transforms (core/multimodal/transforms.py): integer mapping statistics, CenterRoll cost,
# feature-map remap, coverage bookkeeping (csrc/image_transforms.cu)
# --------------------------------------------------------------------------------------------
_PIX_CODES = {torch.int16: 0, torch.int32: 1, torch.int64: 2}


def mapping_image_stats(images, atomic_ptr, pixels, n_img, ref_w=None):
    """Per image: pixel count [n] int64, bbox [n, 4] int32 (x_min, x_max, y_min, y_max; 0 for an image
    without pixels) and, with ref_w, the 256-bin occupancy [n, 8] uint32 of the quantised width
    (core/data_transform/multimodal/image.py:1005).  No synchronisation."""
    require_cuda(images, atomic_ptr, pixels)
    if pixels.dtype not in _PIX_CODES:
        raise TypeError(f"mapping pixels must be int16/int32/int64, got {pixels.dtype}")
    dev = images.device
    images, atomic_ptr, pixels = images.long().contiguous(), atomic_ptr.long().contiguous(), pixels.contiguous()
    count = torch.empty(n_img, dtype=torch.long, device=dev)
    bbox = torch.empty((n_img, 4), dtype=torch.int32, device=dev)
    occ = torch.empty((n_img, 8), dtype=torch.int32, device=dev) if ref_w is not None else None
    launch("dva_mapping_image_stats", dev, images, atomic_ptr, pixels, _PIX_CODES[pixels.dtype], int(images.shape[0]),
           int(n_img), int(ref_w or 0), count, bbox, occ)
    return count, bbox, occ


def center_roll(occ, angular_res, ref_w):
    """Rollings [n] int64 of CenterRoll from the occupancy of mapping_image_stats (image.py:1009-1029)."""
    require_cuda(occ)
    out = torch.empty(occ.shape[0], dtype=torch.long, device=occ.device)
    launch("dva_center_roll", occ.device, occ.contiguous(), int(occ.shape[0]), int(angular_res), int(ref_w), out)
    return out


_REMAP_ELEM = (1, 2, 4)


def _memory_format(x):
    """channels_last when x is channels-last and not also contiguous (C == 1 or H == W == 1), else contiguous"""
    cl = (not x.is_contiguous()) and x.is_contiguous(memory_format=torch.channels_last)
    return torch.channels_last if cl else torch.contiguous_format


def image_remap(x, out_hw=None, rolls=None, offsets=None, flip=False):
    """out[b, :, y, x'] = x[b, :, oy_b + y, (ox_b + (flip ? Wo-1-x' : x') - r_b) mod W] in one copy: the
    per-image torch.roll of update_rollings, the crop of update_cropping and the horizontal flip.  x is
    [B, C, H, W] of 1, 2 or 4-byte elements, NCHW or channels-last; the output keeps x's memory format.
    rolls [B] int64, offsets [B, 2] int64 (ox, oy) on x's device.  No synchronisation."""
    require_cuda(x)
    if x.dim() != 4 or x.element_size() not in _REMAP_ELEM:
        raise TypeError(f"image_remap: expected a 4-D tensor of 1, 2 or 4-byte elements, got {tuple(x.shape)} "
                        f"{x.dtype}")
    B, C, H, W = x.shape
    Ho, Wo = (H, W) if out_hw is None else (int(out_hw[0]), int(out_hw[1]))
    fmt = _memory_format(x)
    x = x.contiguous(memory_format=fmt)
    out = torch.empty((B, C, Ho, Wo), dtype=x.dtype, device=x.device, memory_format=fmt)
    rolls = rolls.to(x.device, torch.long).contiguous() if rolls is not None else None
    offsets = offsets.to(x.device, torch.long).contiguous() if offsets is not None else None
    launch("dva_image_remap", x.device, x, out, B, C, H, W, Ho, Wo, x.element_size(), int(fmt == torch.channels_last),
           rolls, offsets, int(bool(flip)))
    return out


class CoverageIndex:
    """Unseen-point counts of PickImagesFromMemoryCredit (image.py:804-867) without the dense
    bool[n_img, N] table: `gimg` [V] global image id of every view (setting base + local id), `vpoint` [V]
    its point.  `unseen` [n_img] int32 starts at the view count of every image; pick(g) marks g's points
    seen and takes every newly seen point off the count of each image that sees it."""

    def __init__(self, gimg, vpoint, n_img, num_points):
        require_cuda(gimg, vpoint)
        self.dev = gimg.device
        self.V, self.n_img, self.N = int(gimg.shape[0]), int(n_img), int(num_points)
        self.ws = _lib.workspace(_lib.load().dva_coverage_index_workspace_bytes(self.V, self.n_img, self.N), self.dev)
        self.unseen = torch.empty(self.n_img, dtype=torch.int32, device=self.dev)
        self.seen = torch.empty(max(self.N, 1), dtype=torch.int32, device=self.dev)
        self._gimg, self._vpoint = gimg.long().contiguous(), vpoint.long().contiguous()
        launch("dva_coverage_index", self.dev, self._gimg, self._vpoint, self.V, self.n_img, self.N, self.unseen,
               self.seen, self.ws, self.ws.numel())

    def pick(self, g):
        launch("dva_coverage_pick", self.dev, int(g), self.V, self.n_img, self.N, self.unseen, self.seen, self.ws,
               self.ws.numel())


# --------------------------------------------------------------------------------------------
# image loading (SameSettingImageData.read_images, NonStaticMask): Pillow-exact resize and the
# non-static pixel mask (csrc/image_resample.cu)
# --------------------------------------------------------------------------------------------
_PRECISION_BITS = 32 - 8 - 2


def _bicubic(x):
    """Pillow's bicubic_filter (a = -0.5) in float64, with its evaluation order."""
    a = -0.5
    x = np.abs(x)
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def resample_axis_tables(in_size, in0, in1, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for one axis and one box [in0, in1) (C floats):
    bounds [out, 2] int32 (first source index, count) and weights [out, ksize] int32 scaled by 2^22.  Every
    float64 operation is a separate numpy ufunc call, so nothing is fused or reassociated, and the weight sum
    is taken sequentially in source order."""
    span = float(np.float32(in1) - np.float32(in0))             # float subtraction, then (double)
    scale = span / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = float(np.float32(in0)) + (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum(np.trunc(center - support + 0.5).astype(np.int64), 0)
    xmax = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), in_size) - xmin
    j = np.arange(ksize, dtype=np.int64)
    w = _bicubic(((j[None, :] + xmin[:, None]) - center[:, None] + 0.5) * (1.0 / filterscale))
    w = np.where(j[None, :] < xmax[:, None], w, 0.0)
    ww = np.zeros(out_size, dtype=np.float64)
    for k in range(ksize):
        ww = ww + w[:, k]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    scaled = w * float(1 << _PRECISION_BITS)
    k32 = np.trunc(np.where(w < 0, -0.5 + scaled, 0.5 + scaled)).astype(np.int32)
    return np.stack([xmin, xmax], axis=1).astype(np.int32), k32


def _pinned_to(a, device):
    t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    return t.to(device, non_blocking=True)


def image_resample(src, size, boxes=None):
    """PIL.Image.resize(size, box=box) with the BICUBIC filter, bit for bit, on a batch of uint8 images of one
    size: `src` is a [B, C, H, W] uint8 CUDA tensor (any memory format; channels-last avoids a copy) or a list of
    [C, H, W] ones; `size` = (W_out, H_out); `boxes` None (the whole image), (x0, y0, x1, y1) for every image or
    [B, 4] per image, as C floats.  Returns [B, C, H_out, W_out] uint8 in channels-last memory, the layout of
    torch.from_numpy(np.stack(arrays)).permute(0, 3, 1, 2).  The coefficient tables are built on the host and
    uploaded from pinned memory: no synchronisation, unless `boxes` is a CUDA tensor (one device->host read)."""
    if isinstance(src, (list, tuple)):
        src = torch.stack(list(src))
    require_cuda(src)
    if src.dim() != 4 or src.dtype != torch.uint8:
        raise TypeError(f"image_resample: expected a [B, C, H, W] uint8 tensor, got {tuple(src.shape)} {src.dtype}")
    B, C, Hi, Wi = (int(v) for v in src.shape)
    Wo, Ho = int(size[0]), int(size[1])
    if Wo < 1 or Ho < 1:
        raise ValueError(f"image_resample: output size must be positive, got {tuple(size)}")
    bx = np.broadcast_to(np.asarray([0, 0, Wi, Hi] if boxes is None else
                                    (boxes.cpu().numpy() if isinstance(boxes, torch.Tensor) else boxes),
                                    dtype=np.float32), (B, 4))
    if (bx[:, 0] < 0).any() or (bx[:, 1] < 0).any() or (bx[:, 2] > Wi).any() or (bx[:, 3] > Hi).any():
        raise ValueError("image_resample: box can't exceed original image size")
    if (bx[:, 2] <= bx[:, 0]).any() or (bx[:, 3] <= bx[:, 1]).any():
        raise ValueError("image_resample: box can't be empty")
    nhwc = src.permute(0, 2, 3, 1).contiguous()
    out = torch.empty((B, Ho, Wo, C), dtype=torch.uint8, device=src.device)
    # Pillow runs a pass only when that axis changes; an identity pass reproduces the input exactly, so one
    # batch-wide decision per axis gives every image Pillow's bytes
    need_h = bool(((bx[:, 0] != 0) | (bx[:, 2] != Wo)).any()) or Wo != Wi
    need_v = bool(((bx[:, 1] != 0) | (bx[:, 3] != Ho)).any()) or Ho != Hi
    if B == 0 or not (need_h or need_v):
        out.copy_(nhwc)
        return out.permute(0, 3, 1, 2)
    shared = bool((bx == bx[:1]).all())
    rows = bx[:1] if shared else bx

    def tables(n_in, c0, c1, n_out):
        per = [resample_axis_tables(n_in, r[c0], r[c1], n_out) for r in rows]
        k = max(t[1].shape[1] for t in per)
        coef = np.zeros((len(per), n_out, k), dtype=np.int32)
        for i, t in enumerate(per):
            coef[i, :, :t[1].shape[1]] = t[1]
        return np.stack([t[0] for t in per]), coef

    xb, xc = tables(Wi, 0, 2, Wo)
    yb, yc = tables(Hi, 1, 3, Ho)
    yfirst, T = None, Ho
    if need_h and need_v:
        first = yb[:, 0, 0].copy()
        T = int((yb[:, -1, 0] + yb[:, -1, 1] - first).max())
        yb[:, :, 0] -= first[:, None]
        yfirst = np.broadcast_to(first, (B,)).astype(np.int32)
    dev = src.device
    tmp = torch.empty((B, T, Wo, C), dtype=torch.uint8, device=dev) if (need_h and need_v) else None
    d = lambda a: _pinned_to(a, dev)  # noqa: E731
    xb_d, xc_d = (d(xb), d(xc)) if need_h else (None, None)
    yb_d, yc_d = (d(yb), d(yc)) if need_v else (None, None)
    yf_d = d(yfirst) if yfirst is not None else None
    launch("dva_resample_u8", dev, nhwc, tmp, out, B, Hi, Wi, C, Ho, Wo, T, xb_d, xc_d, int(xc.shape[2]),
           int(not shared), yb_d, yc_d, int(yc.shape[2]), int(not shared), yf_d)
    return out.permute(0, 3, 1, 2)


def nonstatic_mask(imgs):
    """[W, H] bool: True where every channel of some image i >= 1 differs from image 0 (NonStaticMask,
    data_transform image.py:139-154).  `imgs` [n, C, H, W] uint8 CUDA, n >= 2.  No synchronisation."""
    require_cuda(imgs)
    if imgs.dim() != 4 or imgs.dtype != torch.uint8 or imgs.shape[0] < 2:
        raise TypeError(f"nonstatic_mask: expected [n >= 2, C, H, W] uint8, got {tuple(imgs.shape)} {imgs.dtype}")
    n, C, H, W = (int(v) for v in imgs.shape)
    nhwc = imgs.permute(0, 2, 3, 1).contiguous()
    mask = torch.empty((W, H), dtype=torch.bool, device=imgs.device)
    launch("dva_nonstatic_mask", imgs.device, nhwc, n, H, W, C, mask)
    return mask


# --------------------------------------------------------------------------------------------
# colour transforms (ColorJitter, ToFloatImage, Normalize): torchvision's tensor arithmetic
# (csrc/image_color.cu)
# --------------------------------------------------------------------------------------------
_JITTER_CODES = {"brightness": 0, "contrast": 1, "saturation": 2}


def color_jitter_u8(x, ops_seq):
    """torchvision's ColorJitter for drawn factors on a [B, 3, H, W] uint8 CUDA tensor (NCHW or channels-last; the
    output keeps x's memory format).  `ops_seq`: the active ops in the drawn order, as (name, factor) pairs with
    name in 'brightness' / 'contrast' / 'saturation'.  The contrast mean is exact (csrc/image_color.cu).  No
    synchronisation."""
    require_cuda(x)
    if x.dim() != 4 or x.shape[1] != 3 or x.dtype != torch.uint8:
        raise TypeError(f"color_jitter_u8: expected a [B, 3, H, W] uint8 tensor, got {tuple(x.shape)} {x.dtype}")
    if len(ops_seq) > 3:
        raise ValueError("color_jitter_u8: at most three ops")
    fmt = _memory_format(x)
    x = x.contiguous(memory_format=fmt)
    out = torch.empty_like(x, memory_format=fmt)
    codes, args = 0, []
    for i, (name, factor) in enumerate(ops_seq):
        codes |= _JITTER_CODES[name] << (4 * i)
        args += [float(factor), float(1.0 - float(factor))]   # 1 - ratio in float64, rounded to fp32 by ctypes
    args += [0.0, 0.0] * (3 - len(ops_seq))
    B, _, H, W = (int(v) for v in x.shape)
    ws = _lib.workspace(_lib.load().dva_color_jitter_u8_workspace_bytes(B), x.device)
    launch("dva_color_jitter_u8", x.device, x, out, B, H, W, int(fmt == torch.channels_last), len(ops_seq), codes,
           *args, ws, ws.numel())
    return out


def image_to_float(x, mean=None, std=None):
    """(x - mean_c) / std_c in fp32 with true division on a [B, C, H, W] CUDA tensor, 1 <= C <= 4, NCHW or
    channels-last (kept).  x uint8 with mean = std = None is ToFloatImage (x.float() / 255 as on the CPU); x fp32
    with per-channel mean / std (sequences of C floats, or of 1 for all channels) is Normalize.  The statistics are
    rounded to fp32 and passed by value: no copy to the device, no synchronisation."""
    require_cuda(x)
    if x.dim() != 4 or x.dtype not in (torch.uint8, torch.float32):
        raise TypeError(f"image_to_float: expected a [B, C, H, W] uint8 or float32 tensor, got {tuple(x.shape)} "
                        f"{x.dtype}")
    C = int(x.shape[1])
    if not 1 <= C <= 4:
        raise TypeError(f"image_to_float: 1 to 4 channels, got {C}")
    if mean is None:
        mean, std = [0.0], [255.0]

    def per_channel(v, what):
        v = [float(a) for a in (v.tolist() if isinstance(v, torch.Tensor) else v)]
        if len(v) == 1:
            v = v * C
        if len(v) != C:
            raise ValueError(f"image_to_float: {what} has {len(v)} values for {C} channels")
        return v + [1.0] * (4 - C)
    m, s = per_channel(mean, "mean"), per_channel(std, "std")
    fmt = _memory_format(x)
    x = x.contiguous(memory_format=fmt)
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device, memory_format=fmt)
    B, _, H, W = (int(v) for v in x.shape)
    launch("dva_image_to_float", x.device, x, int(x.dtype == torch.uint8), out, B, C, H, W,
           int(fmt == torch.channels_last), *m, *s)
    return out


# --------------------------------------------------------------------------------------------
# log-softmax NLL over a view CSR (models/segmentation/multimodal/no3d.py:144-154; csrc/csr_nll.cu)
# --------------------------------------------------------------------------------------------
CSR_NLL_MAX_CLASSES = 64


class _CSRNLLLoss(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, logits, labels, csr_idx, ignore_index):
        V, K = logits.shape
        N = labels.shape[0]
        need_grad = ctx.needs_input_grad[0]
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        stats = torch.empty(3, dtype=torch.int64, device=logits.device)
        lse = torch.empty(V, dtype=torch.float32, device=logits.device) if need_grad else None
        ws = _lib.workspace(_lib.load().dva_csr_nll_fwd_workspace_bytes(N), logits.device)
        launch("dva_csr_nll_fwd", logits.device, logits, dtype_code(logits), labels, csr_idx, V, N, K, int(ignore_index),
               lse, loss, stats, ws, ws.numel())
        _, bad, bad_csr = stats.tolist()
        if bad:
            raise ValueError(f"csr_nll_loss: {bad} view(s) have a label outside [0, {K}) that is not "
                             f"ignore_index={ignore_index}")
        if bad_csr:
            raise ValueError(f"csr_nll_loss: csr_idx must run from 0 to the number of views ({V})")
        ctx.cfg = (V, N, K, int(ignore_index))
        ctx.save_for_backward(logits, labels, csr_idx, lse, stats)
        return loss

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        logits, labels, csr_idx, lse, stats = ctx.saved_tensors
        V, N, K, ignore_index = ctx.cfg
        grad = torch.empty_like(logits)
        g = grad_loss.detach().float().contiguous().view(1)
        launch("dva_csr_nll_bwd", logits.device, logits, dtype_code(logits), labels, csr_idx, V, N, K, ignore_index,
               lse, g, stats, grad)
        return grad, None, None, None


def csr_nll_loss(logits, labels, csr_idx=None, ignore_index=-1):
    """F.nll_loss(F.log_softmax(logits, -1), repeat_interleave(labels, csr_idx.diff()),
    ignore_index=ignore_index) with the mean reduction (no3d.py:144-154), without the [V] target
    and [V, K] log-prob tensors: view v takes the label of its point through the CSR.

    logits [V, K] fp32 / bf16 / fp16 (fp32 math, K <= 64), labels [N] int64, csr_idx [N+1] int64 or
    None for one view per point (V == N, the point-level loss).  Returns a float32 scalar: the mean
    over views whose label is in [0, K) (NaN when there is none, as F.nll_loss); the sum is taken in
    fp64 in a fixed order, so two calls give the same bits.  A label outside [0, K) that is not
    ignore_index raises ValueError (read back after the forward; no device assert)."""
    require_cuda(logits, labels, csr_idx)
    if logits.dim() != 2:
        raise ValueError(f"csr_nll_loss: logits must be [V, K], got shape {tuple(logits.shape)}")
    if logits.dtype not in DTYPE_CODES:
        raise TypeError(f"csr_nll_loss: unsupported logits dtype {logits.dtype}; expected float32/bfloat16/float16")
    V, K = logits.shape
    if not 1 <= K <= CSR_NLL_MAX_CLASSES:
        raise ValueError(f"csr_nll_loss: {K} classes; this kernel supports 1 to {CSR_NLL_MAX_CLASSES}")
    if labels.dim() != 1 or labels.dtype != torch.int64:
        raise TypeError("csr_nll_loss: labels must be a 1D int64 tensor")
    if csr_idx is None:
        if labels.shape[0] != V:
            raise ValueError(f"csr_nll_loss: without csr_idx, labels ({labels.shape[0]}) and logits ({V}) must "
                             f"have one row per point")
    else:
        csr_idx = _check_csr(csr_idx, logits.device)
        if csr_idx.numel() != labels.shape[0] + 1:
            raise ValueError("csr_nll_loss: csr_idx must have one more entry than labels")
    return _CSRNLLLoss.apply(logits.contiguous(), labels.contiguous(), csr_idx, ignore_index)
