"""Autograd operators over the C ABI (include/dva_b200.h).

Each function mirrors one operator of the reference's multimodal path (same argument meaning,
same empty-segment / tie / eps semantics) and is backed ONLY by the sm_90a kernels of
libdva_b200.so: CPU tensors or a missing library raise.  Reference citations are relative to the
reference repository root.
"""
import contextlib
import dataclasses
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
        ggate = torch.empty((2, G), dtype=torch.float32, device=x.device) if gw is not None else None
        # gate-gradient partials and the lane kernel's range queue
        ws = _lib.workspace(_lib.load().dva_view_attention_bwd_workspace_bytes(G), x.device)
        launch("dva_view_attention_bwd", x.device, x, idx, idx64, compat, csr_idx, gw, gb, grad_out, seg_max,
               seg_den, seg_arg, gx_rows, gcompat, ggate, scatter, N, V, R, C, G, int(scaling), dtype_code(x), ws,
               ws.numel())
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
    def forward(ctx, logits, labels, csr_idx, ignore_index, weight):
        V, K = logits.shape
        N = labels.shape[0]
        need_grad = ctx.needs_input_grad[0]
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        stats = torch.empty(3, dtype=torch.int64, device=logits.device)
        lse = torch.empty(V, dtype=torch.float32, device=logits.device) if need_grad else None
        wsum = None
        if weight is None:
            ws = _lib.workspace(_lib.load().dva_csr_nll_fwd_workspace_bytes(N), logits.device)
            launch("dva_csr_nll_fwd", logits.device, logits, dtype_code(logits), labels, csr_idx, V, N, K,
                   int(ignore_index), lse, loss, stats, ws, ws.numel())
        else:
            wsum = torch.empty(1, dtype=torch.float64, device=logits.device)
            ws = _lib.workspace(_lib.load().dva_csr_nll_weighted_fwd_workspace_bytes(N), logits.device)
            launch("dva_csr_nll_weighted_fwd", logits.device, logits, dtype_code(logits), labels, csr_idx, V, N, K,
                   int(ignore_index), weight, lse, loss, wsum, stats, ws, ws.numel())
        _, bad, bad_csr = stats.tolist()
        if bad:
            raise ValueError(f"csr_nll_loss: {bad} view(s) have a label outside [0, {K}) that is not "
                             f"ignore_index={ignore_index}")
        if bad_csr:
            raise ValueError(f"csr_nll_loss: csr_idx must run from 0 to the number of views ({V})")
        ctx.cfg = (V, N, K, int(ignore_index))
        ctx.save_for_backward(logits, labels, csr_idx, lse, stats, weight, wsum)
        return loss

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        logits, labels, csr_idx, lse, stats, weight, wsum = ctx.saved_tensors
        V, N, K, ignore_index = ctx.cfg
        grad = torch.empty_like(logits)
        g = grad_loss.detach().float().contiguous().view(1)
        if weight is None:
            launch("dva_csr_nll_bwd", logits.device, logits, dtype_code(logits), labels, csr_idx, V, N, K,
                   ignore_index, lse, g, stats, grad)
        else:
            launch("dva_csr_nll_weighted_bwd", logits.device, logits, dtype_code(logits), labels, csr_idx, V, N, K,
                   ignore_index, weight, lse, g, wsum, grad)
        return grad, None, None, None, None


def csr_nll_loss(logits, labels, csr_idx=None, ignore_index=-1, weight=None):
    """F.nll_loss(F.log_softmax(logits, -1), repeat_interleave(labels, csr_idx.diff()),
    ignore_index=ignore_index, weight=weight) with the mean reduction (no3d.py:144-154,
    models/segmentation/sparseconv3d.py:41-58), without the [V] target and [V, K] log-prob tensors:
    view v takes the label of its point through the CSR.

    logits [V, K] fp32 / bf16 / fp16 (fp32 math, K <= 64), labels [N] int64, csr_idx [N+1] int64 or
    None for one view per point (V == N, the point-level loss).  Returns a float32 scalar: the mean
    over views whose label is in [0, K) (NaN when there is none, as F.nll_loss); the sum is taken in
    fp64 in a fixed order, so two calls give the same bits.  A label outside [0, K) that is not
    ignore_index raises ValueError (read back after the forward; no device assert).

    weight: optional [K] float32 class weights on the logits' device.  The loss is then
    sum w[y] (lse - x[y]) / sum w[y] over the counted views (NaN when the weights sum to 0, as in
    torch), on separate kernels; weight=None runs the unweighted ones."""
    require_cuda(logits, labels, csr_idx, weight)
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
    if weight is not None:
        if weight.dtype != torch.float32 or weight.dim() != 1 or weight.shape[0] != K:
            raise ValueError(f"csr_nll_loss: weight must be a [{K}] float32 tensor, got {weight.dtype} "
                             f"{tuple(weight.shape)}")
        if weight.device != logits.device:
            raise RuntimeError("csr_nll_loss: weight must live on the device of the logits")
        weight = weight.detach().contiguous()
    return _CSRNLLLoss.apply(logits.contiguous(), labels.contiguous(), csr_idx, ignore_index, weight)


# --------------------------------------------------------------------------------------------
# Lovász-softmax (metrics/lovasz_loss.py:155-230; csrc/lovasz.cu)
# --------------------------------------------------------------------------------------------
LOVASZ_MAX_CLASSES = 64


class _LovaszSoftmax(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, probas, labels, class_mult, present, ignore, log_probs):
        P, K = probas.shape
        dev = probas.device
        keys = torch.empty((K, P), dtype=torch.float32, device=dev)
        launch("dva_lovasz_keys", dev, probas, dtype_code(probas), int(log_probs), labels, P, K, int(ignore), keys)
        # stable, descending: ties keep point order; ignored points (key -1) go after every valid one
        skeys, perm = torch.sort(keys, dim=1, descending=True, stable=True)
        del keys
        need_grad = ctx.needs_input_grad[0]
        fgs = torch.empty((K, P), dtype=torch.uint8, device=dev)
        gsorted = torch.empty((K, P), dtype=torch.float32, device=dev) if need_grad else None
        loss = torch.empty((), dtype=torch.float32, device=dev)
        scale = torch.empty(K, dtype=torch.float32, device=dev)
        ws = _lib.workspace(_lib.load().dva_lovasz_fwd_workspace_bytes(P, K), dev)
        launch("dva_lovasz_fwd", dev, skeys, perm, labels, P, K, class_mult, int(present), fgs, gsorted, loss, scale,
               ws, ws.numel())
        ctx.log_probs = bool(log_probs)
        if need_grad:
            ctx.save_for_backward(probas, skeys, perm, fgs, gsorted, scale)
        return loss

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        probas, skeys, perm, fgs, gsorted, scale = ctx.saved_tensors
        P, K = probas.shape
        grad = torch.empty_like(probas)
        g = grad_loss.detach().float().contiguous().view(1)
        launch("dva_lovasz_bwd", probas.device, probas, dtype_code(probas), int(ctx.log_probs), skeys, perm, fgs,
               gsorted, scale, g, P, K, grad)
        return grad, None, None, None, None, None


def lovasz_softmax(probas, labels, classes="present", ignore=-1, log_probs=False, per_image=False):
    """Multi-class Lovász-softmax loss: lovasz_softmax_flat(*flatten_probas(probas, labels, ignore),
    classes) of metrics/lovasz_loss.py:155-230 for [P, K] inputs (per_image=False).

    probas [P, K] fp32 / bf16 / fp16 class probabilities (fp32 math, 2 <= K <= 64), or
    log-probabilities with log_probs=True (exp taken in the kernel, the gradient chained through it);
    labels [P] int64; points labelled `ignore` are left out.  classes: 'present' (classes with a
    valid point), 'all', or a list of class ids (a repeated id counts twice, as in the reference).
    Returns a float32 scalar, the mean over the kept classes of sum_j e_j g_j (errors sorted
    descending, g the Jaccard differences); fp64 partials in a fixed order, so two calls give the
    same bits.  The sort is torch's stable sort: tied errors are ordered by point index (the
    reference's CPU torch.sort is unstable; the loss does not depend on the order of ties, the
    gradient of one element of a tied block does).  With no valid point, or no kept class, the loss
    is 0 and the gradient 0."""
    if per_image:
        raise NotImplementedError("lovasz_softmax(per_image=True) is not supported")
    require_cuda(probas, labels)
    if probas.dim() != 2:
        raise ValueError(f"lovasz_softmax: probas must be [P, K], got shape {tuple(probas.shape)}")
    if probas.dtype not in DTYPE_CODES:
        raise TypeError(f"lovasz_softmax: unsupported probas dtype {probas.dtype}; expected float32/bfloat16/float16")
    P, K = probas.shape
    if K == 1:
        raise NotImplementedError("lovasz_softmax: the single-class (sigmoid) branch is not supported")
    if not 2 <= K <= LOVASZ_MAX_CLASSES:
        raise ValueError(f"lovasz_softmax: {K} classes; this kernel supports 2 to {LOVASZ_MAX_CLASSES}")
    if labels.dim() != 1 or labels.dtype != torch.int64 or labels.shape[0] != P:
        raise TypeError(f"lovasz_softmax: labels must be a [{P}] int64 tensor")
    if labels.device != probas.device:
        raise RuntimeError("lovasz_softmax: labels must live on the device of probas")
    if isinstance(classes, str):
        if classes not in ("all", "present"):
            raise ValueError(f"lovasz_softmax: classes must be 'all', 'present' or a list, got {classes!r}")
        mult = [1] * K
    else:
        mult = [0] * K
        for c in classes:
            c = int(c)
            if not 0 <= c < K:
                raise ValueError(f"lovasz_softmax: class {c} outside [0, {K})")
            mult[c] += 1
    class_mult = torch.tensor(mult, dtype=torch.int32, device=probas.device)
    return _LovaszSoftmax.apply(probas.contiguous(), labels.contiguous(), class_mult, classes == "present",
                                int(ignore), bool(log_probs))


# ------------------------------------------------------------------------------------------------
# segmentation evaluation (libdva_eval.so, include/dva_eval.h): confusion update, vote accumulation,
# full-resolution nearest-neighbour prediction.  No host read: range errors go to a device status word
# (int32 [1], bits _lib.DVA_EVAL_BAD_*) that the caller reads when it wants the metrics.
# ------------------------------------------------------------------------------------------------
EVAL_MAX_CLASSES = 64
_NN_MODES = {"interpolate": 0, "interpolate_mean": 1, "own_votes": 2}


def eval_status(device):
    """A fresh device status word for the evaluation operators."""
    return torch.zeros(1, dtype=torch.int32, device=device)


def _eval_classes(K, what):
    if not 1 <= K <= EVAL_MAX_CLASSES:
        raise ValueError(f"{what}: {K} classes; the evaluation kernels support 1 to {EVAL_MAX_CLASSES}")


def _ignore_args(ignore_label):
    return (0, 0) if ignore_label is None else (int(ignore_label), 1)


def _check_vec(t, n, dtype, what, name):
    if t.dim() != 1 or t.shape[0] != n or t.dtype != dtype:
        raise TypeError(f"{what}: {name} must be a [{n}] {dtype} tensor, got {tuple(t.shape)} {t.dtype}")


def confusion_update(cm, scores_or_pred, labels, ignore_label=None, counts=None, status=None):
    """cm += the confusion of (labels, prediction) in place: np.bincount(K * gt + argmax(outputs, 1)) of
    metrics/segmentation_tracker.py:76-85 without the host copy.

    cm int64 [K, K] (row = ground truth, column = prediction), K <= 64; scores_or_pred either scores [n, K]
    fp32 / bf16 / fp16, whose argmax is taken in the kernel with numpy's rule (first index of the maximum,
    the first NaN wins), or int64 predictions [n]; labels int64 [n].  Rows labelled `ignore_label` are
    skipped, and with counts (int32 [n], scores only) the rows whose count is 0.  A label (or prediction)
    outside [0, K) is not counted; it sets a bit of `status` (int32 [1]), which is returned."""
    require_cuda(cm, scores_or_pred, labels, counts, status)
    if cm.dim() != 2 or cm.shape[0] != cm.shape[1] or cm.dtype != torch.int64 or not cm.is_contiguous():
        raise TypeError("confusion_update: cm must be a contiguous [K, K] int64 tensor")
    K = cm.shape[0]
    _eval_classes(K, "confusion_update")
    n = scores_or_pred.shape[0]
    _check_vec(labels, n, torch.int64, "confusion_update", "labels")
    status = eval_status(cm.device) if status is None else status
    ign, has_ign = _ignore_args(ignore_label)
    if scores_or_pred.is_floating_point():
        if scores_or_pred.dim() != 2 or scores_or_pred.shape[1] != K:
            raise ValueError(f"confusion_update: scores must be [n, {K}], got {tuple(scores_or_pred.shape)}")
        if counts is not None:
            _check_vec(counts, n, torch.int32, "confusion_update", "counts")
        launch("dva_eval_confusion_scores", cm.device, scores_or_pred.contiguous(), dtype_code(scores_or_pred),
               labels.contiguous(), None if counts is None else counts.contiguous(), n, K, ign, has_ign, cm, status)
    else:
        _check_vec(scores_or_pred, n, torch.int64, "confusion_update", "predictions")
        if counts is not None:
            raise ValueError("confusion_update: counts applies to scores, not to predictions")
        launch("dva_eval_confusion_pred", cm.device, scores_or_pred.contiguous(), labels.contiguous(), n, K, ign,
               has_ign, cm, status)
    return status


def vote(votes, counts, stamp, ids, outputs, status=None):
    """votes[ids] += outputs; counts[ids] += 1 in place (metrics/s3dis_tracker.py:76-80).

    votes fp32 [N, K] (K <= 64), counts int32 [N], stamp int32 [N] all -1 (kept by the caller with the
    table; it is -1 again on return), ids int64 [n], outputs [n, K] fp32 / bf16 / fp16, added in fp32 with one
    rounding per element (torch's votes + outputs).  A duplicated id takes its last occurrence (torch's
    index_put_ leaves it undefined); an id outside [0, N) is skipped and sets a bit of `status`, returned."""
    require_cuda(votes, counts, stamp, ids, outputs, status)
    if votes.dim() != 2 or votes.dtype != torch.float32 or not votes.is_contiguous():
        raise TypeError("vote: votes must be a contiguous [N, K] float32 tensor")
    N, K = votes.shape
    _eval_classes(K, "vote")
    for t, name in ((counts, "counts"), (stamp, "stamp")):
        _check_vec(t, N, torch.int32, "vote", name)
        if not t.is_contiguous():
            raise TypeError(f"vote: {name} must be contiguous")
    n = ids.shape[0]
    _check_vec(ids, n, torch.int64, "vote", "ids")
    if outputs.dim() != 2 or tuple(outputs.shape) != (n, K):
        raise ValueError(f"vote: outputs must be [{n}, {K}], got {tuple(outputs.shape)}")
    status = eval_status(votes.device) if status is None else status
    try:
        launch("dva_eval_vote", votes.device, outputs.contiguous(), dtype_code(outputs), ids.contiguous(), n, N, K,
               votes, counts, stamp, status)
    except RuntimeError:
        stamp.fill_(-1)     # a failed add launch leaves claims behind; a stale claim would drop a later vote
        raise
    return status


def full_res_predict(votes, counts, pos, labels=None, cm=None, ignore_label=None, mode="interpolate", status=None):
    """Full-resolution predictions from a vote table: knn_interpolate(votes[voted], pos[voted], pos, k=1)
    followed by argmax (and the confusion update), fused, without the [N, K] interpolated tensor.

    votes fp32 [N, K], counts int32 [N], pos [N, 3]; voted = the points with counts > 0, in index order.
    The nearest voted point comes from mapping.knn_query (ties to the lower index); the row is weighted in
    torch_geometric's fp32 order.  mode:
      'interpolate'       every point from its nearest voted point (s3dis_tracker.py:94-118);
      'interpolate_mean'  the same, the voted rows divided by their counts first
                          (scannet_segmentation_tracker.py:122-135; the table is not modified);
      'own_votes'         a voted point keeps the argmax of its own votes, the others are interpolated
                          (kitti360_tracker.py:219-222).
    With labels (int64 [N]) and cm (int64 [K, K]) also cm += confusion(labels, pred), skipping
    `ignore_label`.  Returns (pred int64 [N], status)."""
    from .core.multimodal.mapping import knn_query
    require_cuda(votes, counts, pos, labels, cm, status)
    if mode not in _NN_MODES:
        raise ValueError(f"full_res_predict: mode must be one of {sorted(_NN_MODES)}, got {mode!r}")
    if votes.dim() != 2 or votes.dtype != torch.float32 or not votes.is_contiguous():
        raise TypeError("full_res_predict: votes must be a contiguous [N, K] float32 tensor")
    N, K = votes.shape
    _eval_classes(K, "full_res_predict")
    _check_vec(counts, N, torch.int32, "full_res_predict", "counts")
    if pos.dim() != 2 or tuple(pos.shape) != (N, 3):
        raise ValueError(f"full_res_predict: pos must be [{N}, 3], got {tuple(pos.shape)}")
    if (labels is None) != (cm is None):
        raise ValueError("full_res_predict: labels and cm go together")
    if labels is not None:
        _check_vec(labels, N, torch.int64, "full_res_predict", "labels")
        if tuple(cm.shape) != (K, K) or cm.dtype != torch.int64 or not cm.is_contiguous():
            raise TypeError(f"full_res_predict: cm must be a contiguous [{K}, {K}] int64 tensor")
    pos = pos.float().contiguous()
    counts = counts.contiguous()
    has = counts > 0
    voted = torch.nonzero(has).squeeze(1)
    if voted.numel() == 0:
        raise ValueError("full_res_predict: no point has a vote (empty search set)")
    query = torch.arange(N, dtype=torch.int64, device=votes.device)
    if mode == "own_votes":
        unvoted = torch.nonzero(~has).squeeze(1)
        nbr = torch.zeros(N, dtype=torch.int64, device=votes.device)
        nbr[unvoted] = knn_query(pos[unvoted], pos[voted], 1).squeeze(1)
    else:
        nbr = knn_query(pos, pos[voted], 1).squeeze(1)
    status = eval_status(votes.device) if status is None else status
    pred = torch.empty(N, dtype=torch.int64, device=votes.device)
    ign, has_ign = _ignore_args(ignore_label)
    launch("dva_eval_nn_vote", votes.device, votes, counts, pos, N, K, voted, voted.numel(), query, nbr, N,
           _NN_MODES[mode], None if labels is None else labels.contiguous(), ign, has_ign, pred, cm, status)
    return pred, status


# --------------------------------------------------------------------------------------------
# from-scratch image encoder (libdva_conv2d.so, include/dva_conv2d.h): the Conv2dWS -> GroupNorm -> ReLUWS units
# of ResNetDown and ResBlock (modalities/image.py:39-340), each one autograd node.  Maps are channels-last
# [B, H, W, C] fp32; products are 3xTF32 on tensor cores, also under autocast (the inputs are cast to fp32).
# --------------------------------------------------------------------------------------------
RELU_WS_SCALE = math.sqrt(2 / (1 - 1 / math.pi))   # ReLUWS._SCALE (image.py:119)
# (kernel_size, stride, padding) -> convolution kind; the only shapes of the shipped configs
CONV_KINDS = {(3, 1, 1): _lib.DVA_CONV_3X3_REFLECT, (2, 2, 0): _lib.DVA_CONV_2X2_S2, (1, 1, 0): _lib.DVA_CONV_1X1}
_TAPS = {_lib.DVA_CONV_3X3_REFLECT: 3, _lib.DVA_CONV_2X2_S2: 2, _lib.DVA_CONV_1X1: 1}


def conv_out_hw(kind, H, W):
    """Spatial size of a convolution of `kind`, raising ValueError where torch's reflect pad or conv2d raises."""
    if kind != _lib.DVA_CONV_1X1 and (H < 2 or W < 2):
        what = "reflect padding" if kind == _lib.DVA_CONV_3X3_REFLECT else "a 2x2 convolution"
        raise ValueError(f"{what} needs every spatial side >= 2, got {H}x{W}")
    return (H // 2, W // 2) if kind == _lib.DVA_CONV_2X2_S2 else (H, W)


def _conv_weights(w, kind, standardize):
    """(wf, wd): the filter the forward reads ([Co][R][S][Ci]) and the one the data gradient reads."""
    Co, Ci = w.shape[:2]
    wf = torch.empty(w.numel(), dtype=torch.float32, device=w.device)
    wd = torch.empty_like(wf)
    launch("dva_conv2d_weight_prep", w.device, w, Co, Ci, kind, int(standardize), wf, wd)
    return wf, wd


def _weight_grad(w, dwf, kind, standardize):
    if not standardize:     # 1x1: [Co][1][1][Ci] is the torch layout
        return dwf.view_as(w)
    dw = torch.empty_like(w)
    launch("dva_conv2d_weight_prep_bwd", w.device, w, dwf, w.shape[0], w.shape[1], kind, dw)
    return dw


def _conv_fwd(x, wf, bias, Co, kind, G, eps):
    B, H, W, Ci = x.shape
    Ho, Wo = conv_out_hw(kind, H, W)
    z = torch.empty(B, Ho, Wo, Co, dtype=torch.float32, device=x.device)
    mean = torch.empty(B, G, dtype=torch.float32, device=x.device)
    invstd = torch.empty_like(mean)
    ws = _lib.workspace(_lib.load_conv().dva_conv2d_fwd_workspace_bytes(B, Ho, Wo, Co, G), x.device)
    launch("dva_conv2d_fwd", x.device, x, B, H, W, Ci, wf, bias, Co, kind, G, float(eps), z, mean, invstd, ws,
           ws.numel())
    return z, mean, invstd


def _gn_apply(z, gn, relu, skip=None, ds=None):
    """act(GN(z)) [+ skip] [+ GN_ds(z_ds)]; gn = (G, mean, invstd, gamma, beta), ds = (z_ds, G, mean, ...)."""
    B, Ho, Wo, C = z.shape
    G, mean, invstd, gamma, beta = gn
    zs, _, ms, iss, gs, bs = ds if ds is not None else (None,) * 6
    y = torch.empty_like(z)
    launch("dva_conv2d_gn_apply", z.device, z, B, Ho * Wo, C, G, mean, invstd, gamma, beta,
           RELU_WS_SCALE if relu else 0.0, skip, zs, ms, iss, gs, bs, y)
    return y


def _gn_bwd(dy, z, gn, relu):
    B, Ho, Wo, C = z.shape
    G, mean, invstd, gamma, beta = gn
    dz = torch.empty_like(z)
    dgamma = torch.empty(C, dtype=torch.float32, device=z.device)
    dbeta = torch.empty_like(dgamma)
    ws = _lib.workspace(_lib.load_conv().dva_conv2d_gn_bwd_workspace_bytes(B, Ho * Wo, C, G), z.device)
    launch("dva_conv2d_gn_bwd", z.device, dy, z, B, Ho * Wo, C, G, mean, invstd, gamma, beta,
           RELU_WS_SCALE if relu else 0.0, dz, dgamma, dbeta, ws, ws.numel())
    return dz, dgamma, dbeta


def _wgrad(dz, x, kind):
    B, H, W, Ci = x.shape
    Co, T = dz.shape[-1], _TAPS[kind]
    dwf = torch.empty(Co * T * T * Ci, dtype=torch.float32, device=x.device)
    dbias = torch.empty(Co, dtype=torch.float32, device=x.device)
    ws = _lib.workspace(_lib.load_conv().dva_conv2d_wgrad_workspace_bytes(B, H, W, Ci, Co, kind), x.device)
    launch("dva_conv2d_wgrad", x.device, dz, x, B, H, W, Ci, Co, kind, dwf, dbias, ws, ws.numel())
    return dwf, dbias


def _dgrad(dz, x_shape, wd, kind, add=None, out=None):
    """conv^T(dz) [+ add] into out (a new tensor when None; out may be add)."""
    B, H, W, Ci = x_shape
    dx = out if out is not None else torch.empty(B, H, W, Ci, dtype=torch.float32, device=dz.device)
    launch("dva_conv2d_dgrad", dz.device, dz, B, H, W, Ci, dz.shape[-1], wd, kind, add, dx)
    return dx


def _f32(*ts):
    return [None if t is None else t.detach().float().contiguous() for t in ts]


def _rows_input(x, c_in):
    """x as the image kernels read it: channels-last rows [B, H, W, c_in], fp32, contiguous (a copy for any other
    dtype or layout; outside autocast custom_fwd casts nothing)."""
    if x.dim() != 4 or x.shape[3] != c_in:
        raise ValueError(f"expected channels-last rows [B, H, W, {c_in}], got shape {tuple(x.shape)}")
    if not x.is_floating_point():
        raise TypeError(f"expected a floating-point feature map, got {x.dtype}")
    return x.float().contiguous()


def _as_dtypes(grads, dtypes):
    """Each gradient in the dtype of its input (the kernels compute in fp32)."""
    return tuple(None if g is None else g.to(d) for g, d in zip(grads, dtypes))


@dataclasses.dataclass(frozen=True)
class _ConvFamily:
    """The weight-standardised convolutions of one half of the from-scratch image network, as _ConvGNAct and
    _ResBlock call them: k3 is the kind of its 3x3 convolution; weights(w, kind) -> (wf, wd); fwd(x, wf, bias, C_out,
    kind, G, eps) -> (z, mean, invstd); wgrad(dz, x, kind) -> (dwf, dbias); dgrad(dz, x_shape, wd, kind, add=None,
    out=None) -> dx; weight_grad(w, dwf, kind) -> dw; c_in / c_out are the weight dimensions of the input / output
    channels.  (Not a tuple: custom_fwd would rebuild a tuple argument from a generator.)"""
    k3: int
    weights: object
    fwd: object
    wgrad: object
    dgrad: object
    weight_grad: object
    c_in: int
    c_out: int


# the encoder's Conv2dWS: reflect padding, w [C_out][C_in][R][S]
_ENCODER = _ConvFamily(_lib.DVA_CONV_3X3_REFLECT, lambda w, kind: _conv_weights(w, kind, True), _conv_fwd, _wgrad,
                       _dgrad, lambda w, dwf, kind: _weight_grad(w, dwf, kind, True), 1, 0)


class _ConvGNAct(torch.autograd.Function):
    """ReLUWS(GroupNorm(conv(x))) as one node, conv a Conv2dWS (ResNetDown.conv_in, image.py:302-312) or a
    ConvTranspose2dWS (ResNetUp.conv_in) of family `fam`.  Saves x, z and the per-(image, group) statistics."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, x, weight, bias, gamma, beta, kind, G, eps, fam):
        require_cuda(x, weight, bias, gamma, beta)
        ctx.dtypes = [t.dtype for t in (x, weight, bias, gamma, beta)]
        x = _rows_input(x, weight.shape[fam.c_in])
        w, b, g, be = _f32(weight, bias, gamma, beta)
        wf, wd = fam.weights(w, kind)
        z, mean, invstd = fam.fwd(x, wf, b, w.shape[fam.c_out], kind, G, eps)
        ctx.save_for_backward(x, w, wd, g, be, z, mean, invstd)
        ctx.cfg = (kind, G, fam)
        return _gn_apply(z, (G, mean, invstd, g, be), True)

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        x, w, wd, g, be, z, mean, invstd = ctx.saved_tensors
        kind, G, fam = ctx.cfg
        dz, dg, dbe = _gn_bwd(dy.float().contiguous(), z, (G, mean, invstd, g, be), True)
        dwf, db = fam.wgrad(dz, x, kind)
        dx = fam.dgrad(dz, x.shape, wd, kind) if ctx.needs_input_grad[0] else None
        return (*_as_dtypes((dx, fam.weight_grad(w, dwf, kind), db, dg, dbe), ctx.dtypes), None, None, None, None)


class _ResBlock(torch.autograd.Function):
    """ResBlock (image.py:128-189) as one node: h = ReLUWS(GN1(conv1(x))), y = ReLUWS(GN2(conv2(h))) + skip, skip =
    x or GN_ds(conv1x1(x)), the residual added after the second activation.  conv1 and conv2 are the 3x3
    convolutions of family `fam` (Conv2dWS, or ConvTranspose2dWS with stride 1 and zero padding 1); the 1x1
    downsample is a plain nn.Conv2d with bias on libdva_conv2d.so either way.  Saves x, z1, z2, z_ds and the
    statistics; h is recomputed in the backward."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, x, w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed, cfg, fam):
        require_cuda(x, w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed)
        (G1, eps1), (G2, eps2), (Gd, epsd) = cfg
        ctx.dtypes = [None if t is None else t.dtype for t in (x, w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed)]
        x = _rows_input(x, w1.shape[fam.c_in])
        w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed = _f32(w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed)
        k3 = fam.k3
        wf1, wd1 = fam.weights(w1, k3)
        z1, m1, i1 = fam.fwd(x, wf1, b1, w1.shape[fam.c_out], k3, G1, eps1)
        h = _gn_apply(z1, (G1, m1, i1, g1, be1), True)
        wf2, wd2 = fam.weights(w2, k3)
        z2, m2, i2 = fam.fwd(h, wf2, b2, w2.shape[fam.c_out], k3, G2, eps2)
        del h
        ds = None
        wdd = zd = md = idd = None
        if wd is not None:
            wfd, wdd = _conv_weights(wd, _lib.DVA_CONV_1X1, False)
            zd, md, idd = _conv_fwd(x, wfd, bd, wd.shape[0], _lib.DVA_CONV_1X1, Gd, epsd)
            ds = (zd, Gd, md, idd, gd, bed)
        y = _gn_apply(z2, (G2, m2, i2, g2, be2), True, skip=x if ds is None else None, ds=ds)
        ctx.save_for_backward(x, w1, wd1, g1, be1, z1, m1, i1, w2, wd2, g2, be2, z2, m2, i2, wd, wdd, gd, bed, zd,
                              md, idd)
        ctx.cfg = (cfg, fam)
        return y

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        (x, w1, wd1, g1, be1, z1, m1, i1, w2, wd2, g2, be2, z2, m2, i2, wd, wdd, gd, bed, zd, md,
         idd) = ctx.saved_tensors
        ((G1, _), (G2, _), (Gd, _)), fam = ctx.cfg
        k3, k1 = fam.k3, _lib.DVA_CONV_1X1
        dy = dy.float().contiguous()
        gn1, gn2 = (G1, m1, i1, g1, be1), (G2, m2, i2, g2, be2)
        dz2, dg2, dbe2 = _gn_bwd(dy, z2, gn2, True)
        h = _gn_apply(z1, gn1, True)
        dwf2, db2 = fam.wgrad(dz2, h, k3)
        dh = fam.dgrad(dz2, h.shape, wd2, k3)
        del h
        dz1, dg1, dbe1 = _gn_bwd(dh, z1, gn1, True)
        del dh
        dwf1, db1 = fam.wgrad(dz1, x, k3)
        grads_ds = (None,) * 4
        dx = None
        if wd is not None:
            dzd, dgd, dbed = _gn_bwd(dy, zd, (Gd, md, idd, gd, bed), False)
            dwfd, dbd = _wgrad(dzd, x, k1)
            grads_ds = (_weight_grad(wd, dwfd, k1, False), dbd, dgd, dbed)
            if ctx.needs_input_grad[0]:
                dx = _dgrad(dzd, x.shape, wdd, k1)
        if ctx.needs_input_grad[0]:
            dx = fam.dgrad(dz1, x.shape, wd1, k3, add=dy if dx is None else dx, out=dx)
        grads = (dx, fam.weight_grad(w1, dwf1, k3), db1, dg1, dbe1, fam.weight_grad(w2, dwf2, k3), db2, dg2, dbe2,
                 *grads_ds)
        return (*_as_dtypes(grads, ctx.dtypes), None, None)


def _res_block_args(block):
    """The tensors and GroupNorm (num_groups, eps) of a ResBlock, in the order _ResBlock.forward takes them."""
    c1, n1, _, c2, n2, _ = block.block
    ds = block.downsample
    cd, nd = (ds[0], ds[1]) if ds is not None else (None, None)
    cfg = ((n1.num_groups, n1.eps), (n2.num_groups, n2.eps),
           (nd.num_groups, nd.eps) if nd is not None else (1, 1e-5))
    return (c1.weight, c1.bias, n1.weight, n1.bias, c2.weight, c2.bias, n2.weight, n2.bias,
            cd.weight if cd is not None else None, cd.bias if cd is not None else None,
            nd.weight if nd is not None else None, nd.bias if nd is not None else None, cfg)


def conv_gn_relu_ws(x, conv, norm, kind):
    """ReLUWS(norm(conv(x))) for channels-last x [B, H, W, C_in] (conv a Conv2dWS, norm an nn.GroupNorm): fp32
    [B, H', W', C_out], computed from fp32 operands whatever the dtype and layout of x."""
    return _ConvGNAct.apply(x, conv.weight, conv.bias, norm.weight, norm.bias, kind, norm.num_groups, norm.eps,
                            _ENCODER)


def res_block(x, block):
    """A ResBlock on channels-last x [B, H, W, C_in]: fp32 [B, H, W, C_out], computed from fp32 operands whatever the
    dtype and layout of x."""
    return _ResBlock.apply(x, *_res_block_args(block), _ENCODER)


# --------------------------------------------------------------------------------------------
# from-scratch image decoder (libdva_unet.so, include/dva_unet.h): the ConvTranspose2dWS -> GroupNorm -> ReLUWS
# units of ResNetUp and the transposed ResBlocks (modalities/image.py), each one autograd node, and UnaryConv's 1x1
# convolution.  GroupNorm, ReLUWS, the residual and the 1x1 convolutions run on libdva_conv2d.so.  Same rules as
# the encoder: channels-last [B, H, W, C] fp32 maps, 3xTF32 products, inputs cast to fp32 under autocast, gradients
# in each input's dtype.
# --------------------------------------------------------------------------------------------
# (kernel_size, stride, padding) of a zero-padded ConvTranspose2d -> kind; the only shapes of the shipped configs
CONVT_KINDS = {(2, 2, 0): _lib.DVA_UNET_UP_2X2, (3, 1, 1): _lib.DVA_UNET_T_3X3}


def convt_out_hw(kind, H, W):
    """Spatial size of a transposed convolution of `kind` (output_padding 0)."""
    if H < 1 or W < 1:
        raise ValueError(f"a transposed convolution needs a non-empty map, got {H}x{W}")
    return (2 * H, 2 * W) if kind == _lib.DVA_UNET_UP_2X2 else (H, W)


def _convt_weights(w, kind):
    """(wf, wd): the standardised filter as the forward reads it and as the data gradient reads it."""
    Ci, Co = w.shape[:2]
    wf = torch.empty(w.numel(), dtype=torch.float32, device=w.device)
    wd = torch.empty_like(wf)
    launch("dva_unet_weight_prep", w.device, w, Ci, Co, kind, wf, wd)
    return wf, wd


def _convt_weight_grad(w, dwf, kind):
    dw = torch.empty_like(w)
    launch("dva_unet_weight_prep_bwd", w.device, w, dwf, w.shape[0], w.shape[1], kind, dw)
    return dw


def _convt_fwd(x, wf, bias, Co, kind, G, eps):
    B, H, W, Ci = x.shape
    Ho, Wo = convt_out_hw(kind, H, W)
    z = torch.empty(B, Ho, Wo, Co, dtype=torch.float32, device=x.device)
    mean = torch.empty(B, G, dtype=torch.float32, device=x.device)
    invstd = torch.empty_like(mean)
    ws = _lib.workspace(_lib.load_unet().dva_unet_fwd_workspace_bytes(B, H, W, Co, G, kind), x.device)
    launch("dva_unet_fwd", x.device, x, B, H, W, Ci, wf, bias, Co, kind, G, float(eps), z, mean, invstd, ws,
           ws.numel())
    return z, mean, invstd


def _convt_wgrad(dz, x, kind):
    B, H, W, Ci = x.shape
    Co = dz.shape[-1]
    dwf = torch.empty(Ci * Co * (4 if kind == _lib.DVA_UNET_UP_2X2 else 9), dtype=torch.float32, device=x.device)
    dbias = torch.empty(Co, dtype=torch.float32, device=x.device)
    ws = _lib.workspace(_lib.load_unet().dva_unet_wgrad_workspace_bytes(B, H, W, Ci, Co, kind), x.device)
    launch("dva_unet_wgrad", x.device, dz, x, B, H, W, Ci, Co, kind, dwf, dbias, ws, ws.numel())
    return dwf, dbias


def _convt_dgrad(dz, x_shape, wd, kind, add=None, out=None):
    """The data gradient of the transposed convolution [+ add] into out (a new tensor when None; out may be add)."""
    B, H, W, Ci = x_shape
    dx = out if out is not None else torch.empty(B, H, W, Ci, dtype=torch.float32, device=dz.device)
    launch("dva_unet_dgrad", dz.device, dz, B, H, W, Ci, dz.shape[-1], wd, kind, add, dx)
    return dx


# the decoder's ConvTranspose2dWS: zero padding, transposed weights w [C_in][C_out][R][S]
_DECODER = _ConvFamily(_lib.DVA_UNET_T_3X3, _convt_weights, _convt_fwd, _convt_wgrad, _convt_dgrad,
                       _convt_weight_grad, 0, 1)


class _UnaryConv(torch.autograd.Function):
    """UnaryConv's act(conv1x1(x)) (the 1x1 on libdva_conv2d.so, weight-standardised or not; act = relu * scale or
    the identity when scale is 0) as one node.  Saves x and z."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, x, weight, bias, standardize, scale):
        require_cuda(x, weight, bias)
        ctx.dtypes = [t.dtype for t in (x, weight, bias)]
        x = _rows_input(x, weight.shape[1])
        w, b = _f32(weight, bias)
        k1 = _lib.DVA_CONV_1X1
        wf, wd = _conv_weights(w, k1, standardize)
        z, _, _ = _conv_fwd(x, wf, b, w.shape[0], k1, 1, 1e-5)
        ctx.save_for_backward(x, w, wd, z)
        ctx.cfg = (standardize, scale)
        if not scale:
            return z
        y = torch.empty_like(z)
        launch("dva_unet_act", z.device, z, z.numel(), float(scale), y)
        return y

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        x, w, wd, z = ctx.saved_tensors
        standardize, scale = ctx.cfg
        k1 = _lib.DVA_CONV_1X1
        dz = dy.float().contiguous()
        if scale:
            dz_act = torch.empty_like(z)
            launch("dva_unet_act_bwd", z.device, dz, z, z.numel(), float(scale), dz_act)
            dz = dz_act
        dwf, db = _wgrad(dz, x, k1)
        dx = _dgrad(dz, x.shape, wd, k1) if ctx.needs_input_grad[0] else None
        return (*_as_dtypes((dx, _weight_grad(w, dwf, k1, standardize), db), ctx.dtypes), None, None)


def convt_gn_relu_ws(x, conv, norm, kind):
    """ReLUWS(norm(conv(x))) for channels-last x [B, H, W, C_in] (conv a ConvTranspose2dWS, norm an nn.GroupNorm):
    fp32 [B, H', W', C_out], computed from fp32 operands whatever the dtype and layout of x."""
    return _ConvGNAct.apply(x, conv.weight, conv.bias, norm.weight, norm.bias, kind, norm.num_groups, norm.eps,
                            _DECODER)


def res_block_t(x, block):
    """A ResBlock of ConvTranspose2dWS on channels-last x [B, H, W, C_in]: fp32 [B, H, W, C_out], computed from fp32
    operands whatever the dtype and layout of x."""
    return _ResBlock.apply(x, *_res_block_args(block), _DECODER)


def unary_conv(x, conv, standardize, scale):
    """act(conv(x)) for channels-last x [B, H, W, C_in] and a 1x1 conv (nn.Conv2d or Conv2dWS with bias): fp32
    [B, H, W, C_out]; act = relu(.) * scale, or none when scale is 0."""
    return _UnaryConv.apply(x, conv.weight, conv.bias, bool(standardize), float(scale))


# --------------------------------------------------------------------------------------------
# ADE20K ResNet-18 encoder (libdva_resnet.so, include/dva_resnet.h): mit_semseg's resnet18dilated behind the
# reference's ADE20KResNet18* wrappers (modalities/image.py:793-956).  One autograd node per stem unit (conv -> BN ->
# ReLU), per BasicBlock (its hidden activation recomputed in the backward), for the max pool and for a (multi-map)
# bilinear resize.  BatchNorm is F.batch_norm on one device: in training mode the batch statistics normalise and the
# running stats are updated inside the forward (a second call, such as the recompute of a reentrant checkpoint,
# updates them again).  Maps are channels-last [B, H, W, C] fp32; products are 3xTF32 on tensor cores, also under
# autocast (the inputs are cast to fp32); gradients come back in each input's dtype.
# --------------------------------------------------------------------------------------------
def rn_out(n, stride):
    """Output side of a stride-`stride` convolution or max pool of the trunk: ceil(n / stride)."""
    return (n - 1) // stride + 1


def _rn_weights(w):
    """(wf, wd): the filter the forward reads ([Co][T][T][Ci]) and the one the data gradient reads ([Ci][T][T][Co])."""
    Co, Ci, T = w.shape[0], w.shape[1], w.shape[2]
    wf = torch.empty(w.numel(), dtype=torch.float32, device=w.device)
    wd = torch.empty_like(wf)
    launch("dva_resnet_weight_prep", w.device, w, Co, Ci, T, wf, wd)
    return wf, wd


def _rn_running(t):
    """A running-stat buffer as the kernel updates it in place: itself when fp32 and contiguous, else a copy."""
    return t if t.dtype == torch.float32 and t.is_contiguous() else t.detach().float().contiguous()


def _rn_conv_bn(x, wf, Co, geo, bn, sync=None):
    """z = conv(x) and the BatchNorm statistics of z; bn = (running_mean, running_var, training, momentum, eps); sync
    a _BNSync when the statistics are taken over the ranks of a process group."""
    T, stride, dil = geo
    rm, rv, training, momentum, eps = bn
    B, H, W, Ci = x.shape
    Ho, Wo = rn_out(H, stride), rn_out(W, stride)
    z = torch.empty(B, Ho, Wo, Co, dtype=torch.float32, device=x.device)
    mean = torch.empty(Co, dtype=torch.float32, device=x.device)
    invstd = torch.empty_like(mean)
    rm32, rv32 = _rn_running(rm), _rn_running(rv)
    if sync is not None:
        sums = torch.zeros(2 * Co + 1, dtype=torch.float64, device=x.device)
        if B > 0:
            ws = _lib.workspace(_lib.load_resnet().dva_resnet_fwd_workspace_bytes(B, Ho, Wo, Co), x.device)
            launch("dva_resnet_conv_bn_fwd_sums", x.device, x, B, H, W, Ci, wf, Co, T, stride, dil, z, sums, ws,
                   ws.numel())
        sync.count = sync.all_reduce(sums)
        launch("dva_resnet_bn_sync_stats", x.device, sums, Co, sync.count, float(momentum), float(eps), rm32, rv32,
               mean, invstd)
    else:
        ws = _lib.workspace(_lib.load_resnet().dva_resnet_fwd_workspace_bytes(B, Ho, Wo, Co) if training else 0,
                            x.device)
        launch("dva_resnet_conv_bn_fwd", x.device, x, B, H, W, Ci, wf, Co, T, stride, dil, int(training),
               float(momentum), float(eps), rm32, rv32, z, mean, invstd, ws, ws.numel())
    if training:
        for buf, b32 in ((rm, rm32), (rv, rv32)):
            if b32 is not buf:
                buf.copy_(b32)
    return z, mean, invstd


def _rn_apply(z, mean, invstd, gamma, beta, skip=None, ds=None):
    """relu(BN(z) [+ skip] [+ BN_ds(z_ds)]); ds = (z_ds, mean, invstd, gamma, beta)."""
    B, H, W, C = z.shape
    zs, ms, iss, gs, bs = ds if ds is not None else (None,) * 5
    y = torch.empty_like(z)
    if B == 0:      # a rank without images in a synchronised BatchNorm
        return y
    launch("dva_resnet_bn_apply", z.device, z, B * H * W, C, mean, invstd, gamma, beta, skip, zs, ms, iss, gs, bs, y)
    return y


def _rn_bn_bwd(dy, y, z, mean, invstd, gamma, training, want_g=False, sync=None):
    """(dz, g, dgamma, dbeta) of y = relu(BN(z) + r); g, the gradient reaching r, only when want_g.  sync: the
    forward's _BNSync (the sums of g and g * zhat all-reduced over its group; dgamma and dbeta stay this rank's)."""
    B, H, W, C = z.shape
    M = B * H * W
    dz = torch.empty_like(z)
    g = torch.empty_like(z) if want_g else None
    dgamma = torch.empty(C, dtype=torch.float32, device=z.device)
    dbeta = torch.empty_like(dgamma)
    if sync is not None:
        sums = torch.zeros(2 * C + 1, dtype=torch.float64, device=z.device)
        if M > 0:
            ws = _lib.workspace(_lib.load_resnet().dva_resnet_bn_bwd_workspace_bytes(M, C), z.device)
            launch("dva_resnet_bn_bwd_sums", z.device, dy, y, z, M, C, mean, invstd, dgamma, dbeta, sums, ws,
                   ws.numel())
        else:
            dgamma.zero_()
            dbeta.zero_()
        sync.all_reduce(sums)
        if M > 0:
            ws = _lib.workspace(C * 16, z.device)
            launch("dva_resnet_bn_sync_bwd", z.device, dy, y, z, M, C, mean, invstd, gamma, sums, sync.count, dz, g,
                   ws, ws.numel())
        return dz, g, dgamma, dbeta
    ws = _lib.workspace(_lib.load_resnet().dva_resnet_bn_bwd_workspace_bytes(M, C), z.device)
    launch("dva_resnet_bn_bwd", z.device, dy, y, z, M, C, mean, invstd, gamma, int(training), dz, g, dgamma, dbeta,
           ws, ws.numel())
    return dz, g, dgamma, dbeta


def _rn_wgrad(dz, x, Co, geo):
    T, stride, dil = geo
    B, H, W, Ci = x.shape
    if B == 0:
        return torch.zeros(Co, Ci, T, T, dtype=torch.float32, device=x.device)
    dw = torch.empty(Co, Ci, T, T, dtype=torch.float32, device=x.device)
    ws = _lib.workspace(_lib.load_resnet().dva_resnet_wgrad_workspace_bytes(B, H, W, Ci, Co, T, stride, dil), x.device)
    launch("dva_resnet_conv_wgrad", x.device, dz, x, B, H, W, Ci, Co, T, stride, dil, dw, ws, ws.numel())
    return dw


def _rn_dgrad(dz, x_shape, wd, geo, add=None, out=None):
    """conv^T(dz) [+ add] into out (a new tensor when None; out may be add)."""
    T, stride, dil = geo
    B, H, W, Ci = x_shape
    dx = out if out is not None else torch.empty(B, H, W, Ci, dtype=torch.float32, device=dz.device)
    if B == 0:
        return dx
    launch("dva_resnet_conv_dgrad", dz.device, dz, B, H, W, Ci, dz.shape[-1], wd, T, stride, dil, add, dx)
    return dx


class _BNSync:
    """The process group of a training nn.SyncBatchNorm for one forward, and the global count (values per channel
    over the group's ranks) its forward found; the backward reuses the count."""

    def __init__(self, group):
        self.group = group
        self.count = None

    def all_reduce(self, sums):
        """Sums the packed fp64 [2 C + 1] (per-channel sums, then the count) over the group, in place on the current
        stream; returns the global count.  In the forward a count of at most 1 raises ValueError on every rank, as
        each rank decides it from the same all-reduced value."""
        torch.distributed.all_reduce(sums, group=self.group)
        n = int(sums[-1].item()) if self.count is None else self.count
        if n <= 1:
            raise ValueError(f"Expected more than 1 value per channel when training, got {n} over the "
                             f"{torch.distributed.get_world_size(self.group)} ranks of the process group")
        return n


_SYNC_BN = {"split_at_one_rank": False}


@contextlib.contextmanager
def sync_batchnorm_split_at_one_rank():
    """Inside this context a training nn.SyncBatchNorm takes the split (all-reduce) path also in a process group of
    one rank, where it otherwise takes the fused one; both give the same bits.  For tests and measurements."""
    prev = _SYNC_BN["split_at_one_rank"]
    _SYNC_BN["split_at_one_rank"] = True
    try:
        yield
    finally:
        _SYNC_BN["split_at_one_rank"] = prev


def bn_sync_group(bn):
    """The process group whose union batch a BatchNorm normalises over: for a training nn.SyncBatchNorm when
    torch.distributed is initialised and its group (bn.process_group, default the world) has more than one rank;
    None otherwise (eval mode, no process group, one rank, or any other BatchNorm), as torch's SyncBatchNorm
    decides it."""
    if not (isinstance(bn, torch.nn.SyncBatchNorm) and bn.training):
        return None
    dist = torch.distributed
    if not (dist.is_available() and dist.is_initialized()):
        return None
    group = bn.process_group if bn.process_group else dist.group.WORLD
    if dist.get_world_size(group) > 1 or _SYNC_BN["split_at_one_rank"]:
        return group
    return None


def _bn_cfg(bn):
    """(training, momentum, eps) of bn for one forward.  A plain nn.BatchNorm2d (the ImageNet and Cityscapes trunks)
    and an nn.SyncBatchNorm get torch's bookkeeping here, in the module's forward, as _bn_step does it:
    num_batches_tracked += 1 in training (so a reentrant checkpoint's recompute counts twice, as torch's module does)
    and momentum None as the cumulative average.  mit_semseg's SynchronizedBatchNorm2d (steps_counter False) never
    moves its counter."""
    if not getattr(bn, "steps_counter", True):
        return (bn.training, bn.momentum, bn.eps)
    return (bn.training, _bn_step(bn)[2], bn.eps)


def _rn_bn_cfg(bn):
    """(training, momentum, eps, sync) of bn for one forward: _bn_cfg, and a _BNSync when its statistics are
    synchronised over a process group (bn_sync_group), else None."""
    group = bn_sync_group(bn)
    return (*_bn_cfg(bn), _BNSync(group) if group is not None else None)


class _RNConvBNReLU(torch.autograd.Function):
    """relu(BN(conv(x))), a unit of the deep stem, as one node.  Saves x, z, the statistics and the output (the
    ReLU mask)."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, geo, bn_cfg):
        require_cuda(x, weight, gamma, beta)
        ctx.dtypes = [t.dtype for t in (x, weight, gamma, beta)]
        x = _rows_input(x, weight.shape[1])
        w, g, b = _f32(weight, gamma, beta)
        training, momentum, eps, sync = bn_cfg
        wf, wd = _rn_weights(w)
        z, mean, invstd = _rn_conv_bn(x, wf, w.shape[0], geo, (running_mean, running_var, training, momentum, eps),
                                      sync)
        y = _rn_apply(z, mean, invstd, g, b)
        ctx.save_for_backward(x, wd, g, z, mean, invstd, y)
        ctx.cfg = (geo, training, sync, w.shape[0])
        return y

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        x, wd, g, z, mean, invstd, y = ctx.saved_tensors
        geo, training, sync, Co = ctx.cfg
        dz, _, dg, db = _rn_bn_bwd(dy.float().contiguous(), y, z, mean, invstd, g, training, sync=sync)
        dw = _rn_wgrad(dz, x, Co, geo) if ctx.needs_input_grad[1] else None
        dx = _rn_dgrad(dz, x.shape, wd, geo) if ctx.needs_input_grad[0] else None
        return (*_as_dtypes((dx, dw, dg, db), ctx.dtypes), None, None, None, None)


class _RNBasicBlock(torch.autograd.Function):
    """mit_semseg's BasicBlock as one node: h = relu(bn1(conv1(x))), y = relu(bn2(conv2(h)) + r), r = x or
    bn_ds(conv1x1(x)).  Saves x, z1, z2, z_ds, the statistics and y; h is recomputed in the backward."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, x, w1, g1, b1, w2, g2, b2, wd, gd, bd, rm1, rv1, rm2, rv2, rmd, rvd, cfg):
        require_cuda(x, w1, g1, b1, w2, g2, b2, wd, gd, bd)
        (stride, dil1, dil2), bn1, bn2, bnd = cfg
        ctx.dtypes = [None if t is None else t.dtype for t in (x, w1, g1, b1, w2, g2, b2, wd, gd, bd)]
        x = _rows_input(x, w1.shape[1])
        w1, g1, b1, w2, g2, b2, wd, gd, bd = _f32(w1, g1, b1, w2, g2, b2, wd, gd, bd)
        geo1, geo2, geod = (3, stride, dil1), (3, 1, dil2), (1, stride, 1)
        wf1, wd1 = _rn_weights(w1)
        z1, m1, i1 = _rn_conv_bn(x, wf1, w1.shape[0], geo1, (rm1, rv1, *bn1[:3]), bn1[3])
        h = _rn_apply(z1, m1, i1, g1, b1)
        wf2, wd2 = _rn_weights(w2)
        z2, m2, i2 = _rn_conv_bn(h, wf2, w2.shape[0], geo2, (rm2, rv2, *bn2[:3]), bn2[3])
        del h
        wdd = zd = md = idd = None
        if wd is not None:
            wfd, wdd = _rn_weights(wd)
            zd, md, idd = _rn_conv_bn(x, wfd, wd.shape[0], geod, (rmd, rvd, *bnd[:3]), bnd[3])
            y = _rn_apply(z2, m2, i2, g2, b2, ds=(zd, md, idd, gd, bd))
        else:
            y = _rn_apply(z2, m2, i2, g2, b2, skip=x)
        ctx.save_for_backward(x, wd1, g1, b1, z1, m1, i1, wd2, g2, z2, m2, i2, wdd, gd, zd, md, idd, y)
        ctx.cfg = (geo1, geo2, geod, bn1, bn2, bnd if bnd is not None else (False, None, None, None), w1.shape[0])
        return y

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        x, wd1, g1, b1, z1, m1, i1, wd2, g2, z2, m2, i2, wdd, gd, zd, md, idd, y = ctx.saved_tensors
        geo1, geo2, geod, bn1, bn2, bnd, Co = ctx.cfg
        need = ctx.needs_input_grad
        dy = dy.float().contiguous()
        dz2, gr, dg2, db2 = _rn_bn_bwd(dy, y, z2, m2, i2, g2, bn2[0], want_g=zd is None, sync=bn2[3])
        h = _rn_apply(z1, m1, i1, g1, b1)
        dw2 = _rn_wgrad(dz2, h, Co, geo2) if need[4] else None
        dh = _rn_dgrad(dz2, h.shape, wd2, geo2)
        dz1, _, dg1, db1 = _rn_bn_bwd(dh, h, z1, m1, i1, g1, bn1[0], sync=bn1[3])
        del h, dh
        dw1 = _rn_wgrad(dz1, x, Co, geo1) if need[1] else None
        grads_ds = (None,) * 3
        dx = None
        if zd is not None:
            dzd, _, dgd, dbd = _rn_bn_bwd(dy, y, zd, md, idd, gd, bnd[0], sync=bnd[3])
            grads_ds = (_rn_wgrad(dzd, x, Co, geod) if need[7] else None, dgd, dbd)
            if need[0]:
                dx = _rn_dgrad(dzd, x.shape, wdd, geod)
        if need[0]:
            dx = _rn_dgrad(dz1, x.shape, wd1, geo1, add=gr if dx is None else dx, out=dx)
        grads = (dx, dw1, dg1, db1, dw2, dg2, db2, *grads_ds)
        return (*_as_dtypes(grads, ctx.dtypes), *([None] * 7))


def rn_pool_out(n, padding=1):
    """Output side of the stems' MaxPool2d(3, 2, padding), padding 1 (ceil(n / 2)) or 0 (floor((n - 3) / 2) + 1);
    ValueError when n + 2 padding < 3 leaves no window."""
    if padding not in (0, 1):
        raise ValueError(f"max pool padding must be 0 or 1, got {padding!r}")
    if n + 2 * padding < 3:
        raise ValueError(f"MaxPool2d(3, 2, {padding}): input side {n} is smaller than one window")
    return (n + 2 * padding - 3) // 2 + 1


class _RNMaxPool(torch.autograd.Function):
    """MaxPool2d(3, stride 2, padding 1 or 0) with the window position of the max saved for the backward."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, x, padding):
        require_cuda(x)
        ctx.dtype = x.dtype
        x = x.float().contiguous()
        B, H, W, C = x.shape
        y = torch.empty(B, rn_pool_out(H, padding), rn_pool_out(W, padding), C, dtype=torch.float32, device=x.device)
        arg = torch.empty(y.shape, dtype=torch.uint8, device=x.device)
        if B > 0:
            launch("dva_resnet_maxpool_pad", x.device, x, B, H, W, C, padding, y, arg)
        ctx.save_for_backward(arg)
        ctx.cfg = (B, H, W, C, padding)
        ctx.mark_non_differentiable(arg)
        return y

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        (arg,) = ctx.saved_tensors
        B, H, W, C, padding = ctx.cfg
        dx = torch.empty(B, H, W, C, dtype=torch.float32, device=dy.device)
        if B > 0:
            launch("dva_resnet_maxpool_pad_bwd", dy.device, dy.float().contiguous(), arg, B, H, W, C, padding, dx)
        return dx.to(ctx.dtype), None


def resize_scale(n_in, n_out, scale_factor=None):
    """The scale of torch's bilinear source index (align_corners=False): float32(1 / scale_factor) when a factor is
    given, float32(n_in) / n_out when a size is."""
    if scale_factor is not None and scale_factor > 0:
        return float(np.float32(1.0 / scale_factor))
    return float(np.float32(n_in) / np.float32(n_out))


class _RNResize(torch.autograd.Function):
    """Bilinear resizes (align_corners=False) of several maps [B, H_i, W_i, C_i] to one size, concatenated along the
    channels: each map is written into its own column slice of the [B, Ho, Wo, sum C_i] output."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, size, scales, *xs):
        require_cuda(*xs)
        Ho, Wo = size
        ctx.dtypes = [x.dtype for x in xs]
        xs = [x.float().contiguous() for x in xs]
        B, ld = xs[0].shape[0], sum(x.shape[3] for x in xs)
        y = torch.empty(B, Ho, Wo, ld, dtype=torch.float32, device=xs[0].device)
        col = 0
        for x, (sh, sw) in zip(xs, scales):
            _, H, W, C = x.shape
            if B > 0:
                launch("dva_resnet_resize", x.device, x, B, H, W, C, Ho, Wo, sh, sw, y, ld, col)
            col += C
        ctx.shapes = [tuple(x.shape) for x in xs]
        ctx.cfg = (size, scales, ld)
        return y

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        (Ho, Wo), scales, ld = ctx.cfg
        dy = dy.float().contiguous()
        grads, col = [], 0
        for (B, H, W, C), (sh, sw), need in zip(ctx.shapes, scales, ctx.needs_input_grad[2:]):
            if need:
                dx = torch.empty(B, H, W, C, dtype=torch.float32, device=dy.device)
                if B > 0:
                    launch("dva_resnet_resize_bwd", dy.device, dy, ld, col, B, H, W, C, Ho, Wo, sh, sw, dx)
                grads.append(dx)
            else:
                grads.append(None)
            col += C
        return (None, None, *_as_dtypes(grads, ctx.dtypes))


def rn_conv_bn_relu(x, conv, bn):
    """relu(bn(conv(x))) for channels-last x [B, H, W, C_in] (conv an nn.Conv2d without bias, bn a BatchNorm2d):
    fp32 [B, H', W', C_out]; in training mode bn's running stats are updated."""
    geo = (conv.kernel_size[0], conv.stride[0], conv.dilation[0])
    return _RNConvBNReLU.apply(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, geo,
                               _rn_bn_cfg(bn))


def rn_basic_block(x, block):
    """A BasicBlock (conv1, bn1, conv2, bn2, downsample) on channels-last x [B, H, W, C_in]: fp32 [B, H', W', C_out]."""
    ds = block.downsample
    cd, nd = (ds[0], ds[1]) if ds is not None else (None, None)
    cfg = ((block.conv1.stride[0], block.conv1.dilation[0], block.conv2.dilation[0]), _rn_bn_cfg(block.bn1),
           _rn_bn_cfg(block.bn2), _rn_bn_cfg(nd) if nd is not None else None)
    return _RNBasicBlock.apply(x, block.conv1.weight, block.bn1.weight, block.bn1.bias, block.conv2.weight,
                               block.bn2.weight, block.bn2.bias, cd.weight if cd is not None else None,
                               nd.weight if nd is not None else None, nd.bias if nd is not None else None,
                               block.bn1.running_mean, block.bn1.running_var, block.bn2.running_mean,
                               block.bn2.running_var, nd.running_mean if nd is not None else None,
                               nd.running_var if nd is not None else None, cfg)


def rn_maxpool(x, padding=1):
    """MaxPool2d(3, 2, padding) of channels-last x [B, H, W, C], padding 1 (the ADE20K and ImageNet stems) or 0 (the
    Cityscapes stem): fp32 [B, rn_pool_out(H, padding), rn_pool_out(W, padding), C]."""
    return _RNMaxPool.apply(x, padding)


# --------------------------------------------------------------------------------------------
# The pyramid-pooling head of ADE20KResNet18PPM (modalities/image.py:658-716, PPMFeatMap): for each pool scale s,
# adaptive average pool to s x s -> 1x1 conv -> BatchNorm -> ReLU -> bilinear resize back to h x w; the map and the
# resized branches concatenated, then conv_last (3x3 conv -> BatchNorm -> ReLU).  All on existing kernels: the pool is
# the mean gather pool of libdva_b200.so over an index of torch's bins, the rest libdva_resnet.so.
# --------------------------------------------------------------------------------------------
_PPM_INDEX = {}


def _ppm_index(B, h, w, scales, device):
    """The gather-pool index of the adaptive average pools at `scales` of a [B, h, w, C] map, built on the device and
    cached per shape: one atom per (scale, image, bin), scale-major, so that the pooled rows of scale s are one
    [B, s, s, C] block; an atom's pixels (x, y) are torch's bin [floor(i h / s), ceil((i + 1) h / s)) x
    [floor(j w / s), ceil((j + 1) w / s)), row-major (bins overlap and repeat where s does not divide the side).
    Returns (img [B * sum s^2] int64, pix [P, 2] int32, aptr int64, row offset of each scale)."""
    key = (B, h, w, tuple(scales), str(device))
    if key in _PPM_INDEX:
        return _PPM_INDEX[key]
    imgs, pixs, counts, offsets, off = [], [], [], [], 0
    for s in scales:
        i = torch.arange(s, device=device)
        y0, y1 = (i * h) // s, ((i + 1) * h + s - 1) // s
        x0, x1 = (i * w) // s, ((i + 1) * w + s - 1) // s
        dy = torch.arange(int((y1 - y0).max()), device=device)
        dx = torch.arange(int((x1 - x0).max()), device=device)
        # [bin row, bin col, dy, dx] -> the pixels of each bin, row-major
        y = (y0[:, None, None, None] + dy[None, None, :, None]).expand(s, s, dy.numel(), dx.numel())
        x = (x0[None, :, None, None] + dx[None, None, None, :]).expand(s, s, dy.numel(), dx.numel())
        keep = ((dy[None, None, :, None] < (y1 - y0)[:, None, None, None])
                & (dx[None, None, None, :] < (x1 - x0)[None, :, None, None]))
        pix = torch.stack([x[keep], y[keep]], dim=1).int()
        n = ((y1 - y0)[:, None] * (x1 - x0)[None, :]).reshape(-1)
        pixs.append(pix.repeat(B, 1))
        counts.append(n.repeat(B))
        imgs.append(torch.arange(B, device=device).repeat_interleave(s * s))
        offsets.append(off)
        off += B * s * s
    counts = torch.cat(counts)
    aptr = torch.zeros(counts.numel() + 1, dtype=torch.int64, device=device)
    torch.cumsum(counts, 0, out=aptr[1:])
    idx = (torch.cat(imgs).long().contiguous(), torch.cat(pixs).contiguous(), aptr, offsets)
    _PPM_INDEX[key] = idx
    return idx


def ppm_branch_training(bn, B, s):
    """Whether a pyramid branch's BatchNorm uses batch statistics: PrudentSynchronizedBatchNorm2d runs in eval mode
    for a (1, C, 1, 1) input, so the scale-1 branch at batch size 1 never does; an nn.SyncBatchNorm converted from
    it has no such rule."""
    if isinstance(bn, torch.nn.SyncBatchNorm):
        return bool(bn.training)
    return bool(bn.training) and not (B == 1 and s == 1)


class _RNPPMHead(torch.autograd.Function):
    """PPMFeatMap on channels-last conv5 [B, h, w, C] as one node, with the final resize to out_size.  The concat
    [B, h, w, C + 512 n] is one buffer: conv5 is copied into its first C columns and each branch is resized into its
    own column slice.  Saves the concat, the pooled maps, the pre-activations, statistics and outputs of the five
    BatchNorms and the data-gradient filters.  The pool's backward is the deterministic gather-pool backward, whatever
    torch.use_deterministic_algorithms says: no sum of the head uses atomics."""

    @staticmethod
    @_fwd_f32
    def forward(ctx, x, out_size, scales, branch_cfg, last_cfg, *params):
        require_cuda(x, *params)
        ctx.dtypes = [x.dtype] + [p.dtype for p in params]
        B, h, w, C = x.shape
        x = _rows_input(x, C)
        n = len(scales)
        ws_, gs, bs = _f32(*params[0:3 * n:3]), _f32(*params[1:3 * n:3]), _f32(*params[2:3 * n:3])
        w_last, g_last, b_last = _f32(*params[3 * n:3 * n + 3])
        running = params[3 * n + 3:]
        dev = x.device
        img, pix, aptr, offsets = _ppm_index(B, h, w, scales, dev)
        Vw, P = img.numel(), pix.shape[0]
        pooled = torch.empty(Vw, C, dtype=torch.float32, device=dev)
        if B > 0:       # B == 0: a rank without images in synchronised BatchNorms
            launch("dva_gather_pool_fwd", dev, x, 1, img, pix, 0, aptr, pooled, None, B, C, h, w, Vw, P,
                   REDUCE_CODES["mean"], dtype_code(x))
        ld = C + sum(wk.shape[0] for wk in ws_)
        cat = torch.empty(B, h, w, ld, dtype=torch.float32, device=dev)
        cat[..., :C].copy_(x)
        saved, col = [], C
        for k, s in enumerate(scales):
            xs = pooled[offsets[k]:offsets[k] + B * s * s].view(B, s, s, C)
            wf, wd = _rn_weights(ws_[k])
            Co = ws_[k].shape[0]
            z, mean, invstd = _rn_conv_bn(xs, wf, Co, (1, 1, 1), (running[2 * k], running[2 * k + 1],
                                                                 *branch_cfg[k][:3]), branch_cfg[k][3])
            y = _rn_apply(z, mean, invstd, gs[k], bs[k])
            sh, sw = resize_scale(s, h), resize_scale(s, w)
            if B > 0:
                launch("dva_resnet_resize", dev, y, B, s, s, Co, h, w, sh, sw, cat, ld, col)
            saved += [wd, z, mean, invstd, y]
            col += Co
        wf, wd = _rn_weights(w_last)
        z, mean, invstd = _rn_conv_bn(cat, wf, w_last.shape[0], (3, 1, 1), (running[2 * n], running[2 * n + 1],
                                                                           *last_cfg[:3]), last_cfg[3])
        y = _rn_apply(z, mean, invstd, g_last, b_last)
        out = y
        if out_size is not None:
            out = torch.empty(B, *out_size, y.shape[3], dtype=torch.float32, device=dev)
        if out_size is not None and B > 0:
            launch("dva_resnet_resize", dev, y, B, h, w, y.shape[3], out_size[0], out_size[1],
                   resize_scale(h, out_size[0]), resize_scale(w, out_size[1]), out, y.shape[3], 0)
        ctx.save_for_backward(pooled, cat, *gs, g_last, wd, z, mean, invstd, y, *saved)
        ctx.cfg = (B, h, w, C, tuple(scales), offsets, branch_cfg, last_cfg, out_size)
        return out

    @staticmethod
    @_bwd
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        B, h, w, C, scales, offsets, branch_cfg, last_cfg, out_size = ctx.cfg
        n = len(scales)
        pooled, cat, *rest = ctx.saved_tensors
        gs, g_last, rest = rest[:n], rest[n], rest[n + 1:]
        wd, z, mean, invstd, y = rest[:5]
        branches = [rest[5 + 5 * k:10 + 5 * k] for k in range(n)]
        need = ctx.needs_input_grad[5:]
        dev = dy.device
        dy = dy.float().contiguous()
        Co = y.shape[3]
        if out_size is not None:
            dyh = torch.empty_like(y)
            if B > 0:
                launch("dva_resnet_resize_bwd", dev, dy, Co, 0, B, h, w, Co, out_size[0], out_size[1],
                       resize_scale(h, out_size[0]), resize_scale(w, out_size[1]), dyh)
            dy = dyh
        dz, _, dg_last, db_last = _rn_bn_bwd(dy, y, z, mean, invstd, g_last, last_cfg[0], sync=last_cfg[3])
        dw_last = _rn_wgrad(dz, cat, Co, (3, 1, 1)) if need[3 * n] else None
        dcat = _rn_dgrad(dz, cat.shape, wd, (3, 1, 1))
        del dz
        ld = cat.shape[3]
        dpooled = torch.empty_like(pooled) if ctx.needs_input_grad[0] else None
        grads, col = [], C
        for k, s in enumerate(scales):
            wdk, zk, mk, ik, yk = branches[k]
            Ck = yk.shape[3]
            dyk = torch.empty_like(yk)
            if B > 0:
                launch("dva_resnet_resize_bwd", dev, dcat, ld, col, B, s, s, Ck, h, w, resize_scale(s, h),
                       resize_scale(s, w), dyk)
            dzk, _, dgk, dbk = _rn_bn_bwd(dyk, yk, zk, mk, ik, gs[k], branch_cfg[k][0], sync=branch_cfg[k][3])
            xs = pooled[offsets[k]:offsets[k] + B * s * s].view(B, s, s, C)
            dwk = _rn_wgrad(dzk, xs, Ck, (1, 1, 1)) if need[3 * k] else None
            if dpooled is not None:
                dxs = dpooled[offsets[k]:offsets[k] + B * s * s].view(B, s, s, C)
                _rn_dgrad(dzk, xs.shape, wdk, (1, 1, 1), out=dxs)
            grads += [dwk, dgk, dbk]
            col += Ck
        dx = None
        if dpooled is not None and B == 0:
            dx = dcat[..., :C].clone()
        elif dpooled is not None:
            img, pix, aptr, _ = _ppm_index(B, h, w, scales, dev)
            Vw, P = img.numel(), pix.shape[0]
            dx = torch.empty(B, h, w, C, dtype=torch.float32, device=dev)
            ws = _lib.workspace(_lib.load().dva_gather_pool_bwd_det_workspace_bytes(B, h, w, P), dev)
            launch("dva_gather_pool_bwd_det", dev, dpooled, 1, img, pix, 0, aptr, None, dx, B, C, h, w, Vw, P,
                   REDUCE_CODES["mean"], dtype_code(dpooled), ws, ws.numel())
            dx += dcat[..., :C]
        grads += [dw_last, dg_last, db_last]
        dx, *grads = _as_dtypes([dx] + grads, ctx.dtypes)
        n_running = len(ctx.needs_input_grad) - 5 - len(grads)
        return (dx, None, None, None, None, *grads, *([None] * n_running))


def rn_ppm_head(x, decoder, out_size=None):
    """PPMFeatMap (`decoder`: .ppm[i] = (adaptive pool, 1x1 conv, Prudent BatchNorm, ReLU), .conv_last = (3x3 conv,
    BatchNorm, ReLU)) on channels-last conv5 x [B, h, w, C]: fp32 [B, h, w, 512], or [B, *out_size, 512] after a
    size-based bilinear resize.  Training-mode BatchNorms update their running stats; the scale-1 branch at batch
    size 1 runs in eval mode (ppm_branch_training)."""
    B = x.shape[0]
    scales = [int(m[0].output_size if isinstance(m[0].output_size, int) else m[0].output_size[0])
              for m in decoder.ppm]
    conv, bn = decoder.conv_last[0], decoder.conv_last[1]
    params, running, branch_cfg = [], [], []
    for m, s in zip(decoder.ppm, scales):
        params += [m[1].weight, m[2].weight, m[2].bias]
        running += [m[2].running_mean, m[2].running_var]
        branch_cfg.append((ppm_branch_training(m[2], B, s), *_rn_bn_cfg(m[2])[1:]))
    params += [conv.weight, bn.weight, bn.bias]
    running += [bn.running_mean, bn.running_var]
    size = None if out_size is None else (int(out_size[0]), int(out_size[1]))
    return _RNPPMHead.apply(x, size, scales, branch_cfg, _rn_bn_cfg(bn), *params, *running)


def rn_resize(xs, size, scale_factor=None):
    """Bilinear resizes (align_corners=False) of the channels-last maps xs to size (Ho, Wo), concatenated along the
    channels; scale_factor, when given, sets torch's source scale 1 / scale_factor (F.interpolate(scale_factor=))."""
    scales = [(resize_scale(x.shape[1], size[0], scale_factor), resize_scale(x.shape[2], size[1], scale_factor))
              for x in xs]
    return _RNResize.apply(tuple(int(s) for s in size), scales, *xs)
