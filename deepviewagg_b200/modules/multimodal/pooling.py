"""Drop-in mirror of torch_points3d/modules/multimodal/pooling.py on the sm_90a kernels.

Same class names, constructor kwargs (unknown kwargs are swallowed: the model factory always
injects `index`, unet.py:633-636), `forward(x_main, x_mod, x_map, csr_idx)` signatures,
parameter names/shapes (state_dicts interchange with the reference) and `save_last` taps.
What differs is the execution: the chain

    segment_softmax_csr -> x_mod * expand_group_feat(a) -> segment_csr(sum) -> Gating(segment max)

(pooling.py:285-300 / 515-530) is ONE fused kernel pair (ops.view_attention, optionally with the
upstream row gather of modules.py:518 folded in through `row_index`), every remaining
segment_csr / gather_csr call goes to libdva_b200.so, and the MLPs are library GEMMs.
"""
import math
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from ...core.common_modules import MLP
from ...ops import segment_csr, segment_softmax_csr, gather_csr, segment_gather_csr  # noqa: F401

_local_modules = sys.modules[__name__]

__all__ = [
    "BimodalCSRPool", "HeuristicBimodalCSRPool", "GroupBimodalCSRPool", "QKVBimodalCSRPool",
    "MinMaxDiffSetFeat", "DeepSetFeat", "MLPSetFeat", "Gating", "nearest_power_of_2",
    "group_sizes", "expand_group_feat", "segment_softmax_csr", "gather_csr", "segment_gather_csr",
]


def _dense_index(csr_idx):
    """Point id of every view: arange(N).repeat_interleave(counts), built on the device
    (the reference builds the arange on the host, pooling.py:781, 835)."""
    n = csr_idx.shape[0] - 1
    return torch.arange(n, device=csr_idx.device).repeat_interleave(csr_idx[1:] - csr_idx[:-1])


class _SaveLast:
    """`save_last` debugging / view-loss taps shared by the pools (pooling.py:45-51, 64-70)."""

    def _init_taps(self, save_last, extra=()):
        self.save_last = save_last
        for name in ("x_map", "x_mod", "idx", "view_num") + tuple(extra):
            setattr(self, "_last_" + name, None)

    def _tap_common(self, x_map, x_mod, csr_idx):
        self._last_x_map = x_map
        self._last_x_mod = x_mod
        self._last_idx = _dense_index(csr_idx)
        self._last_view_num = csr_idx[1:] - csr_idx[:-1]


class BimodalCSRPool(nn.Module, _SaveLast):
    """max / mean / min / sum pooling over CSR groups (pooling.py:14-71)."""

    _POOLING_MODES = ['max', 'mean', 'min', 'sum']

    def __init__(self, mode='max', save_last=False, **kwargs):
        super().__init__()
        assert mode in self._POOLING_MODES, \
            f"Unsupported mode '{mode}'. Expected one of: {self._POOLING_MODES}"
        self._mode = mode
        self._init_taps(save_last)

    def forward(self, x_main, x_mod, x_map, csr_idx):
        x_pool = segment_csr(x_mod, csr_idx, reduce=self._mode)
        if self.save_last:
            self._tap_common(x_map, x_mod, csr_idx)
        return x_pool


class HeuristicBimodalCSRPool(nn.Module, _SaveLast):
    """Pick, per point, the view whose mapping feature `feat` is max/min (pooling.py:74-156)."""

    _MODES = ['max', 'min']
    _FEATURES = ['normalized_depth', 'linearity', 'planarity', 'scattering',
                 'orientation_to_the_surface', 'normalized_pixel_height', 'density', 'occlusion']

    def __init__(self, mode='max', feat=0, save_last=False, **kwargs):
        super().__init__()
        assert mode in self._MODES, f"Unsupported mode '{mode}'. Expected one of: {self._MODES}."
        self._mode = mode
        feat = self._FEATURES.index(feat) if isinstance(feat, str) else feat
        assert feat < len(self._FEATURES), \
            f"Feat={feat} is too large. Expected feat<{len(self._FEATURES)}."
        self._feat = feat
        self._init_taps(save_last)

    def forward(self, x_main, x_mod, x_map, csr_idx):
        x_pool = ops.heuristic_pool(x_mod, x_map, csr_idx, self._feat, self._mode)
        if self.save_last:
            self._tap_common(x_map, x_mod, csr_idx)
        return x_pool

    def extra_repr(self) -> str:
        return f'mode={self._mode}, feat={self._FEATURES[self._feat]}, save_last={self.save_last}'


def _attend(x_mod, compat, csr_idx, num_groups, out_mod, gate, group_scaling, row_index=None,
            row_index_is_permutation=False):
    """softmax over views -> weighted sum -> gating. Fused kernel when G is a power of two <= 32,
    otherwise the same chain composed from the unfused CUDA operators.
    Returns (x_pool, attentions, gating or None)."""
    if ops.fused_groups_supported(num_groups):
        gw = gate.weight if gate is not None else None
        gb = gate.bias if gate is not None else None
        if gate is not None and (gw is None or gb is None):  # Gating(weight=False / bias=False)
            gw = gw if gw is not None else torch.ones(1, num_groups, device=compat.device)
            gb = gb if gb is not None else torch.zeros(1, num_groups, device=compat.device)
        x_pool, att, seg_max = ops.view_attention(
            x_mod, compat, csr_idx, num_groups, idx=row_index, gate_weight=gw, gate_bias=gb,
            group_scaling=group_scaling, idx_is_permutation=bool(row_index is not None and row_index_is_permutation))
        gating = None
        if gate is not None:
            with torch.no_grad():
                gating = torch.tanh(F.relu(seg_max * gw.detach().view(1, -1) + gb.detach().view(1, -1)))
                gating = gating.view(-1, num_groups).squeeze(1)
        return x_pool, att, gating
    if row_index is not None:
        x_mod = x_mod[row_index.long()]
    attentions = segment_softmax_csr(compat, csr_idx, scaling=group_scaling)
    x_pool = segment_csr(x_mod * expand_group_feat(attentions, num_groups, out_mod), csr_idx, reduce='sum')
    gating = None
    if gate is not None:
        gating = gate(segment_csr(compat, csr_idx, reduce='max'))
        x_pool = x_pool * expand_group_feat(gating, num_groups, out_mod)
    return x_pool, attentions, gating


def _biased_linear(lin, x):
    """nn.Linear with bias on [rows, K] CUDA fp32 inputs: the projection goes through ops.linear
    (skinny exact-fp32 kernels for K, N <= 64 -- E_score 32 -> G, Q / K 32 -> G*D), the bias is a
    broadcast add; same parameters (`weight`, `bias`) as the reference's nn.Linear."""
    if x.dim() == 2 and ops.tc_gemm_supported(x, lin.weight):
        z = ops.linear(x, lin.weight)
        return z if lin.bias is None else z + lin.bias
    return lin(x)


class GroupBimodalCSRPool(nn.Module, _SaveLast):
    """View attention from mapping features only (the paper's model; pooling.py:159-319).

    forward accepts an optional `row_index` (LongTensor [V]): x_mod is then the un-sorted
    concatenation of per-setting view features and row_index the CSR-friendly order
    (ImageData.view_cat_sorting); the gather is folded into the attention kernel instead of the
    [V,C] copy of modules.py:518.  E_mod is row-wise (its BatchNorm statistics are permutation
    invariant), so E_mod(x)[idx] == E_mod(x[idx]).  `row_index_is_permutation=True` (set by
    UnimodalBranch, where view_cat_sorting is a permutation by construction) lets the backward write
    each x_mod gradient row exactly once; any other row_index (duplicates, subsets) takes the
    accumulating path.
    """

    def __init__(self, in_map=None, in_mod=None, out_mod=None, num_groups=1, use_mod=False,
                 gating=True, group_scaling=True, save_last=False, nc_inner=32,
                 map_encoder='DeepSetFeat', **kwargs):
        super().__init__()
        self.nc_inner = nc_inner
        self._init_taps(save_last, ("C", "A", "G"))
        assert 1 <= num_groups <= in_mod, f"Number of groups must be between 1 and in_mod={in_mod}."
        out_mod = in_mod if out_mod is None else out_mod
        self.in_mod, self.out_mod = in_mod, out_mod
        self.use_mod, self.num_groups, self.group_scaling = use_mod, num_groups, group_scaling
        self.E_map = getattr(_local_modules, map_encoder)(in_map, nc_inner, **kwargs)
        self.E_mod = MLP([in_mod, out_mod, out_mod], bias=False)
        if self.use_mod:
            in_mix, out_mix = nc_inner + out_mod, nc_inner
            mid_mix = nearest_power_of_2((in_mix + out_mix) / 2, out_mix * 2)
            self.E_mix = MLP([in_mix, mid_mix, out_mix], bias=False)
        self.E_score = nn.Linear(nc_inner, num_groups, bias=True)
        self.G = Gating(num_groups, bias=True) if gating else None

    def forward(self, x_main, x_mod, x_map, csr_idx, row_index=None, row_index_is_permutation=False):
        x_map = self.E_map(x_map, csr_idx)
        x_mod = self.E_mod(x_mod)
        if self.use_mod:
            x_rows = x_mod if row_index is None else x_mod[row_index.long()]
            compatibilities = _biased_linear(self.E_score, self.E_mix(torch.cat([x_map, x_rows], dim=1)))
        else:
            compatibilities = _biased_linear(self.E_score, x_map)
        x_pool, attentions, gating = _attend(x_mod, compatibilities, csr_idx, self.num_groups,
                                             self.out_mod, self.G, self.group_scaling, row_index,
                                             row_index_is_permutation)
        if self.save_last:
            self._tap_common(x_map, x_mod if row_index is None else x_mod[row_index.long()], csr_idx)
            self._last_C, self._last_A = compatibilities, attentions
            if self.G:
                self._last_G = gating
        return x_pool

    def extra_repr(self) -> str:
        return "\n".join(f'{a}={getattr(self, a)}'
                         for a in ['num_groups', 'use_mod', 'group_scaling', 'save_last'])


class QKVBimodalCSRPool(nn.Module, _SaveLast):
    """Query (3D point) x key (viewing conditions) attention (pooling.py:322-551)."""

    def __init__(self, in_main=None, in_map=None, in_mod=None, out_mod=None, num_groups=1,
                 use_mod_q=False, use_mod_k=False, nc_qk=8, gating=True, dim_scaling=True,
                 group_scaling=False, debug=False, save_last=False, nc_inner=32,
                 map_encoder='DeepSetFeat', **kwargs):
        super().__init__()
        if debug:
            raise NotImplementedError(
                "QKVBimodalCSRPool(debug=True) draws random inputs inside forward "
                "(pooling.py:463-468) and is not supported")
        self.nc_inner = nc_inner
        self._init_taps(save_last, ("Q", "K", "C", "A", "G"))
        self.debug = False
        assert 1 <= num_groups <= in_mod, f"Number of groups must be between 1 and in_mod={in_mod}."
        out_mod = in_mod if out_mod is None else out_mod
        self.in_mod, self.out_mod, self.nc_qk = in_mod, out_mod, nc_qk
        self.use_mod_q, self.use_mod_k, self.num_groups = use_mod_q, use_mod_k, num_groups
        self.dim_scaling, self.group_scaling = dim_scaling, group_scaling
        self.E_main = MLP([in_main, nc_inner, nc_inner], bias=False)
        self.E_map = getattr(_local_modules, map_encoder)(in_map, nc_inner, **kwargs)
        self.E_mod = MLP([in_mod, out_mod, out_mod], bias=False)
        if self.use_mod_q:
            in_mix, out_mix = nc_inner + out_mod, nc_inner
            self.E_mix_Q = MLP([in_mix, nearest_power_of_2((in_mix + out_mix) / 2, out_mix * 2), out_mix],
                               bias=False)
        self.Q = nn.Linear(nc_inner, nc_qk * num_groups, bias=True)
        if self.use_mod_k:
            in_mix, out_mix = nc_inner + in_mod, nc_inner  # NB in_mod, like pooling.py:442
            self.E_mix_K = MLP([in_mix, nearest_power_of_2((in_mix + out_mix) / 2, out_mix * 2), out_mix],
                               bias=False)
        self.K = nn.Linear(nc_inner, nc_qk * num_groups, bias=True)
        self.G = Gating(num_groups, bias=True) if gating else None

    def forward(self, x_main, x_mod, x_map, csr_idx, row_index=None, row_index_is_permutation=False):
        x_main = self.E_main(x_main)
        x_map = self.E_map(x_map, csr_idx)
        x_mod = self.E_mod(x_mod)
        need_rows = self.use_mod_k or self.use_mod_q
        x_rows = x_mod if (row_index is None or not need_rows) else x_mod[row_index.long()]
        if self.use_mod_k:
            keys = _biased_linear(self.K, self.E_mix_K(torch.cat([x_map, x_rows], dim=1)))
        else:
            keys = _biased_linear(self.K, x_map)
        if self.use_mod_q:
            x_main_q = gather_csr(x_main, csr_idx, n_items=x_map.shape[0])
            queries = _biased_linear(self.Q, self.E_mix_Q(torch.cat([x_main_q, x_rows], dim=1)))
            # one query per view: every view is its own segment for the ragged dot kernel
            view_ptr = torch.arange(keys.shape[0] + 1, device=keys.device)
            compatibilities = ops.qk_scores(keys, queries, view_ptr, self.num_groups, self.dim_scaling)
        else:
            queries = _biased_linear(self.Q, x_main)  # N x (D x num_groups); never expanded to views
            compatibilities = ops.qk_scores(keys, queries, csr_idx, self.num_groups, self.dim_scaling)
        x_pool, attentions, gating = _attend(x_mod, compatibilities, csr_idx, self.num_groups,
                                             self.out_mod, self.G, self.group_scaling, row_index,
                                             row_index_is_permutation)
        if self.save_last:
            self._tap_common(x_map, x_mod if row_index is None else x_mod[row_index.long()], csr_idx)
            self._last_K = keys
            self._last_Q = queries if self.use_mod_q else gather_csr(queries, csr_idx, n_items=keys.shape[0])
            self._last_C, self._last_A = compatibilities, attentions
            if self.G:
                self._last_G = gating
        return x_pool

    def extra_repr(self) -> str:
        return "\n".join(f'{a}={getattr(self, a)}' for a in ['dim_scaling', 'group_scaling', 'save_last'])


class MinMaxDiffSetFeat(nn.Module):
    """Element-wise set features from difference-to-min / -max / set size (pooling.py:554-601)."""

    def __init__(self, d_in, d_out, use_min=True, use_max=True, use_num=False, **kwargs):
        super().__init__()
        self.d_in, self.d_out = d_in, d_out
        self.use_min, self.use_max, self.use_num = use_min, use_max, use_num
        self.mlp = MLP([d_in * (1 + self.use_min + self.use_max) + self.use_num, d_out, d_out], bias=False)

    def forward(self, x, csr_idx):
        parts = [x]
        if self.use_min:
            parts.append(x - segment_gather_csr(x, csr_idx, reduce='min'))
        if self.use_max:
            parts.append(x - segment_gather_csr(x, csr_idx, reduce='max'))
        if self.use_num:
            counts = csr_idx[1:] - csr_idx[:-1]
            num = torch.sqrt(1 / (counts + 1e-3))
            parts.append(gather_csr(num.view(-1, 1).to(x.dtype), csr_idx, n_items=x.shape[0]))
        return self.mlp(torch.cat(parts, dim=1))

    def extra_repr(self) -> str:
        return "\n".join(f'{a}={getattr(self, a)}' for a in ['use_min', 'use_max', 'use_num'])


class DeepSetFeat(nn.Module):
    """DeepSets-style set encoder of the mapping features (pooling.py:604-673)."""

    _POOLING_MODES = ['max', 'mean', 'min', 'sum']
    _FUSION_MODES = ['residual', 'concatenation', 'both']

    def __init__(self, d_in, d_out, pool='max', fusion='concatenation', use_num=False, **kwargs):
        super().__init__()
        pool = pool.split('_')
        assert all(p in self._POOLING_MODES for p in pool), \
            f"Unsupported pool='{pool}'. Expected elements of: {self._POOLING_MODES}"
        if fusion not in self._FUSION_MODES:
            raise NotImplementedError(
                f"Unknown fusion='{fusion}'. Please choose among supported modes: {self._FUSION_MODES}.")
        self.pool, self.fusion = pool, fusion
        self.d_in, self.d_out, self.use_num = d_in, d_out, use_num
        self.mlp_elt_1 = MLP([d_in, d_out, d_out], bias=False)
        self.mlp_set = MLP([d_out * len(self.pool) + self.use_num, d_out, d_out], bias=False)
        self.mlp_elt_2 = MLP([d_out if fusion == 'residual' else d_out * 2, d_out, d_out], bias=False)

    def forward(self, x, csr_idx):
        x = self.mlp_elt_1(x)
        x_set = torch.cat([segment_csr(x, csr_idx, reduce=p) for p in self.pool], dim=-1)
        if self.use_num:
            set_num = torch.sqrt(1 / (csr_idx[1:] - csr_idx[:-1] + 1e-3))
            x_set = torch.cat((x_set, set_num.view(-1, 1).to(x_set.dtype)), dim=1)
        x_set = self.mlp_set(x_set)
        x_set = gather_csr(x_set, csr_idx, n_items=x.shape[0])
        if self.fusion == 'residual':
            x_out = x + x_set
        elif self.fusion == 'concatenation':
            x_out = torch.cat((x, x_set), dim=-1)
        else:
            x_out = torch.cat((x, x + x_set), dim=-1)
        return self.mlp_elt_2(x_out)

    def extra_repr(self) -> str:
        return "\n".join(f'{a}={getattr(self, a)}' for a in ['pool', 'fusion', 'use_num'])


class MLPSetFeat(nn.Module):
    """Set-agnostic element encoder (pooling.py:676-687)."""

    def __init__(self, d_in, d_out, **kwargs):
        super().__init__()
        self.d_in, self.d_out = d_in, d_out
        self.mlp = MLP([d_in, d_out, d_out], bias=False)

    def forward(self, x, csr_idx):
        return self.mlp(x)


class Gating(nn.Module):
    """Rectified-tanh gating with learnable linear correction (pooling.py:690-715).

    Like the reference it updates its input in place (pooling.py:705-711)."""

    def __init__(self, num_groups, weight=True, bias=True, activation='tanh+'):
        super().__init__()
        self.num_groups = num_groups
        self.weight = nn.Parameter(torch.ones(1, num_groups)) if weight else None
        self.bias = nn.Parameter(torch.zeros(1, num_groups)) if bias else None
        if activation not in ('tanh+', 'sigmoid'):
            raise ValueError(f"Activation '{activation}' not supported for Gating")

    def forward(self, x):
        if self.weight is not None:
            x *= self.weight
        if self.bias is not None:
            x += self.bias
        return torch.tanh(F.relu(x, inplace=True)).view(-1, self.num_groups).squeeze(1)

    def extra_repr(self) -> str:
        return f'num_groups={self.num_groups}, weight={self.weight is not None}, bias={self.bias is not None}'


def nearest_power_of_2(x, min_power=16):
    """Nearest power of two of x, not below min_power (pooling.py:718-734)."""
    x = int(x)
    if x < min_power:
        return min_power
    hi = 1 << (x - 1).bit_length()
    lo = hi >> 1
    return lo if x - lo < hi - x else hi


def group_sizes(num_elements, num_groups):
    """Channels per group, as even as possible, wider groups first (pooling.py:737-745)."""
    base, rem = divmod(num_elements, num_groups)
    return torch.tensor([base + (g < rem) for g in range(num_groups)], dtype=torch.long)


def expand_group_feat(A, num_groups, num_channels):
    """Broadcast per-group values to the channels of each group (pooling.py:748-755)."""
    if num_groups == 1:
        A = A.view(-1, 1)
    elif num_groups < num_channels:
        A = A.repeat_interleave(group_sizes(num_channels, num_groups).to(A.device), dim=1)
    return A
