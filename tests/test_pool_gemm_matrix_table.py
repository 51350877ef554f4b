"""Kernel matrix of the feature-map pools (gather_pool.cu), the fused BatchNorm + LeakyReLU (bn_act.cu) and the
projection GEMMs (skinny_gemm.cu, tc_gemm.cu, mlp_layer.cu): the case table, the inputs that route to each case,
the float64 references and their per-element error bounds.

tests/test_gpu_pool_gemm_matrix.py runs every case on the GPU and records, by name, which kernel ran.  This file
checks, without a GPU, that
  * the case table holds exactly the instantiations of these families compiled into libdva_b200.so
    (cuobjdump -symbols), so a new instantiation without a case fails here.  The bucket-sort internals the
    deterministic pool backward uses (bk::count_keys, bk::scatter_keys, the scans, order_by_id) are shared
    with the mapping build and the deterministic row scatter and stay out of this table;
  * every bound can fail: plausible bugs injected into the float64 references break them.

Notation: u32 = 2^-24, u_s = half an ulp of the storage type, K = 8, ke = K u32, tiny = the storage type's smallest
step (2^-126, or 2^-24 for fp16 subnormals).  Every quantity comes from float64 on the exact stored inputs.

Feature-map pools (v_p = the fp32 value of pixel slot p: the stored map element, or the fp32 bilinear sample of
image_oracle.sparse_interpolation_pixels, which follows the kernel's operation order; n = pixels of the view):
  max / min    bit-equal to round_to(T) of the fp32 extreme of the view (exact: rounding is monotone); one-pixel
               views of every reduce bit-equal to round_to(T) of v_p; empty views exactly 0
  sum          u_s |ref| + ke n sum |v_p| + tiny;   mean: the same divided by n
  map gradient (atomic): the contributions c (float(dy), divided by n for the mean, times the fp32 corner weight
               for interp; max / min: only the first arg-extreme slot) are exact fp32 values; their float64
               scatter is the reference, with bound ke (cnt + 1) sum |c| + u_s |ref| + tiny, cnt = contributions
               to the element
  map gradient (deterministic): bit-equal to deterministic_oracle.map_grad_ordered rounded to T.

BatchNorm + LeakyReLU(s) on z [R, C] (VEC = 16 / sizeof(T), or 1 on the scalar path; G = reduce grid =
min(ceil(R / 64), 4 * 132) CTAs, RG = 256 / min(C / VEC, 256) row groups per CTA, L = ceil(ceil(R / G) / RG) + RG + 2
the longest fp32 chain of a column sum; z0 = row 0, the shift of the statistics pass; S1 = sum |z - z0|,
S2 = sum (z - z0)^2; dzin = error of z when it comes out of a GEMM, else 0):
  training  dmu = ke (L S1 / R + |mu|) + mean(dzin),  dvar = ke L (S2 + 2 |mu - z0| S1) / R + 2 mean(|z - mu| dzin),
            dinv = inv (dvar / (2 (var + eps)) + ke)
  eval      dmu = 0, dinv = ke inv (the running statistics are exact inputs)
  pre-activation a = gamma zhat + beta:  da = |gamma| (inv (dmu + dzin) + |z - mu| dinv) + ke (|gamma| inv (|z| + |mu|) + |beta|)
  y         da + u_s |y| + tiny; an element with |a| <= da may take either slope: + (1 - s) |a|  ("flipped")
  d beta    ke L sum |g| + F0,   d gamma  ke L sum |g zhat| + sum |g| dzh + F1,   g = dy act'(a),
            dzh = inv (dmu + dzin) + |z - mu| dinv + ke |zhat|,  F0 = sum_flipped (1 - s) |dy|,  F1 = the same times |zhat|
  dz        (training) dsc |q| + |sc| ((1 - s) |dy| [flipped] + d beta / R + |zhat| d gamma / R + |k1| dzh
            + ke (|g| + |k0| + |zhat k1|)) + u_s |dz| + tiny,  sc = gamma inv, dsc = |gamma| dinv + ke |sc|,
            k0 = d beta / R, k1 = d gamma / R, q = g - k0 - zhat k1;  (eval) k0 = k1 = 0
  running   m dmu + ke |rm'|,  m dvar R / (R - 1) + ke |rv'|.
Statistics from the wgmma rows kernel's epilogue (ops.linear_bn_act in training, dva_linear_bnstats_fwd): CTA b
takes the 128-row tiles b, b + ctas, ... (ctas = min(tiles, 132)) and shifts every column by sh_b = row 0 of its first
tile; a warp sums d = z - sh_b and d^2 over its 16 rows of a tile in fp32 (an add chain of at most 5), the tiles and
warps of the CTA are added in fp64, the CTA's two sums are stored as fp32 (one rounding each), and
bn_stats_finalize_kernel undoes the shifts in fp64: S = sum_b (s_b + n_b sh_b), Q = sum_b (q_b + 2 sh_b s_b + n_b sh_b^2).
With ds_b = 17 ke sum_b |d| + u32 |s_b| and dq_b = (17 ke + u32) q_b (17 >= 5 adds + the rounding of d, with margin):
  dS = sum_b ds_b,  dQ = sum_b (dq_b + 2 |sh_b| ds_b),  dmu = dS / R + ke |mu| + mean(dzin),
  dvar = dQ / R + 2 |mu| dS / R + 2^-50 mean(z^2) (fp64 rounding of Q / R - mu^2) + 2 mean(|z - mu| dzin);
the backward's column sums still come from bn_bwd_reduce_kernel and keep L above.

Projection GEMMs (3xTF32: the split products hi hi + hi lo + lo hi in fp32 accumulators):
  per element (ke (L + 2) + 2^-20) sum_k |a_k b_k| + tiny.  2^-20 covers the dropped lo lo product and the
  truncated lo operands (each <= 2^-22 |a b|); 1xTF32 errs by up to 2^-11 |a b|.  L is the longest fp32
  accumulation chain of the kernel that ran: the reduction length (padded K, or the N outputs for dX) for the rows
  kernels; for dW the rows one CTA accumulates plus the number of CTA partials summed after it, both from the
  launch's grid (dw_chain below).
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import deterministic_oracle as DO
from oracle import image_oracle as IO
from oracle import pooling_oracle as O
from oracle.scatter_standin import segment_csr as S_segment_csr
from test_kernel_matrix_table import (CPP, DTYPES, K_ERR, TINY, U32, U_S, V16, _lib_path, kname,
                                      library_kernels, parse_kernel, ptr_of, round_to, violations)
import test_kernel_matrix_table as KM

KE = K_ERR * U32
NUM_SMS = 132
RED_NAMES = ("sum", "mean", "max", "min")
PIX_CPP = {"i16": "short", "i32": "int"}
PIX_DT = {"i16": torch.int16, "i32": torch.int32}
SLOPE = 0.2

FAMILIES = ("gather_pool_fwd_kernel", "gather_pool_bwd_kernel", "gather_pool_fwd_cl_kernel",
            "gather_pool_bwd_cl_kernel", "det::gather_pool_bwd_det_cl_kernel", "det::gather_pool_bwd_det_kernel",
            "det::describe_entries", "det::slot_views_kernel", "transpose_last2_kernel",
            "bn_stats_kernel", "bn_apply_kernel", "bn_bwd_reduce_kernel", "bn_bwd_apply_kernel", "bn_finalize_kernel",
            "bn_bwd_finalize_kernel",
            "skinny_rows_mma_kernel", "skinny_dw_mma_kernel", "skinny_rows_kernel", "skinny_dw_kernel",
            "skinny_dw_reduce_cols_kernel", "skinny_dw_reduce_kernel",
            "tc::tc_rows_kernel", "tc::tc_dw_kernel", "tc::dw_reduce_kernel", "tc::split_weight_kernel",
            "tc::bn_stats_finalize_kernel", "mlp_layer_bwd_kernel", "mlp_dw_reduce_kernel")


def canonical(name):
    return KM.canonical(name, FAMILIES)


# ------------------------------------------------------------------------------------------------
# feature-map pools: configurations and the kernels each one launches
# ------------------------------------------------------------------------------------------------
# route -> chunks per row (cv = C / VEC) of the channels-last vector kernels: LPR 4, 8, 16, 32 from with_lpr; 3 and
# 40 are not powers of two (idle lanes past the last chunk), 40 needs two LPR-32 tiles
LPR_CV = {4: 3, 8: 8, 16: 12, 32: 40}
POOL_ROUTES = ("nchw", "cl_scalar", "lpr4", "lpr8", "lpr16", "lpr32")


def pool_geometry(route, dt):
    """Map shape and channels of a route.  nchw: few pixels per map pixel (below _NCHW_TRANSPOSE_SHARE), read in
    place; nchw_t: many, so the map is transposed to channels-last; cl_scalar: C not a multiple of VEC;
    cl_misaligned: a channels-last map one element off 16-byte alignment."""
    V = V16[dt]
    if route == "nchw":
        return dict(B=2, H=32, W=48, C=2 * V, cl=False, off=0)
    if route == "nchw_t":
        return dict(B=2, H=8, W=12, C=LPR_CV[16] * V, cl=False, off=0)
    if route == "cl_scalar":
        return dict(B=2, H=12, W=16, C=2 * V + 1, cl=True, off=0)
    if route == "cl_misaligned":
        return dict(B=2, H=12, W=16, C=2 * V, cl=True, off=1)
    return dict(B=2, H=12, W=16, C=LPR_CV[int(route[3:])] * V, cl=True, off=0)


def pool_launches(conf):
    """Every table kernel the configuration (dtype, pixel type, route, reduce, interp) must launch: forward,
    atomic backward, deterministic backward (+ its index kernels, + the transpositions)."""
    dt, pix, route, red, interp = conf
    T, PX = CPP[dt], PIX_CPP[pix]
    ks = {kname("det::describe_entries", PX, interp), "det::slot_views_kernel"}
    if route in ("nchw", "cl_scalar"):
        cl = route == "cl_scalar"
        ks |= {kname("gather_pool_fwd_kernel", T, PX, cl, red, interp),
               kname("gather_pool_bwd_kernel", T, PX, cl, red, interp),
               kname("det::gather_pool_bwd_det_kernel", T, cl, red, interp)}
        return ks
    if route == "cl_misaligned":      # only the forward reads the map; the gradients are fresh, aligned tensors
        lpr = 4
        ks.add(kname("gather_pool_fwd_kernel", T, PX, True, red, interp))
    else:
        lpr = 16 if route == "nchw_t" else int(route[3:])
        ks.add(kname("gather_pool_fwd_cl_kernel", T, PX, lpr, red, interp))
    ks |= {kname("gather_pool_bwd_cl_kernel", T, PX, lpr, red, interp),
           kname("det::gather_pool_bwd_det_cl_kernel", T, lpr, red, interp)}
    if route == "nchw_t":
        ks.add(kname("transpose_last2_kernel", "float" if dt == "f32" else "unsigned short"))
    return ks


def _pool_confs():
    confs = [(dt, pix, route, red, interp) for dt in DTYPES for pix in PIX_CPP for route in POOL_ROUTES
             for red in range(4) for interp in (False, True)]
    for dt in DTYPES:
        confs.append((dt, "i32", "nchw_t", 2, False))
        confs.append((dt, "i32", "nchw_t", 1, True))
        confs.append((dt, "i16", "cl_misaligned", 0, False))
    return confs


POOL_CONFS = _pool_confs()


def _pool_cases():
    """One case per instantiation, owned by the first configuration that launches it."""
    owner = {}
    for conf in POOL_CONFS:
        for k in sorted(pool_launches(conf)):
            owner.setdefault(k, conf)
    return [dict(kind="pool", kernel=k, conf=c) for k, c in owner.items()]


# ------------------------------------------------------------------------------------------------
# BatchNorm + LeakyReLU: per (dtype, vector width) a list of configurations over the edges
# ------------------------------------------------------------------------------------------------
def bn_configs(dt, vec):
    """dict(R, C, training, affine, momentum (None: cumulative average), z_off, special (constant / 1e3-offset
    columns)).  vec > 1: C a multiple of VEC, aligned rows; vec == 1: C = 33 / 1 / 301, or a misaligned z."""
    V = V16[dt]
    wide = 1032 if dt == "f32" else 2056              # C / VEC = 258 / 257 > 256 threads: two column passes
    base = dict(affine=True, momentum=0.1, z_off=0, special=False)
    if vec > 1:
        cs = [dict(R=1000, C=4 * V, training=True, special=True), dict(R=1, C=4 * V, training=False),
              dict(R=2, C=2 * V, training=True, affine=False, momentum=None), dict(R=300, C=wide, training=True),
              dict(R=517, C=V, training=False, special=True)]
    else:
        cs = [dict(R=1000, C=33, training=True, special=True), dict(R=1, C=1, training=False),
              dict(R=2, C=1, training=True, affine=False, momentum=None),
              dict(R=700, C=4 * V, training=True, z_off=1), dict(R=300, C=301, training=True),
              dict(R=50, C=33, training=False, affine=False)]
    return [dict(base, **c) for c in cs]


def bn_launches(dt, vec, training):
    T = CPP[dt]
    ks = {kname("bn_apply_kernel", T, vec), kname("bn_bwd_reduce_kernel", T, vec), "bn_bwd_finalize_kernel",
          kname("bn_bwd_apply_kernel", T, vec)}
    if training:
        ks |= {kname("bn_stats_kernel", T, vec), kname("bn_finalize_kernel", T)}
    return ks


def _bn_cases():
    cases, owned = [], set()
    for dt in DTYPES:
        for vec in (V16[dt], 1):
            for k in sorted(bn_launches(dt, vec, True) - owned):
                cases.append(dict(kind="bn", kernel=k, dtype=dt, vec=vec))
                owned.add(k)
    return cases


# ------------------------------------------------------------------------------------------------
# projection GEMMs: shapes (M, K in, N out, storage offset of x) run through ops.linear forward + backward
# ------------------------------------------------------------------------------------------------
# skinny (K, N <= 64 and not a wgmma shape: N >= 32, K >= 8, both multiples of 4 for the rows GEMMs; N > 32 and
# K > 32 for dW).  Rows kernels: NT from the output width (<= 8 / 16 / 32 / 64); dX has OUT = K in, RED = N out.
# dW tiles (MT, NT): MT = 2 when N out <= 32 (64-column K blocks) else 4 (32-column blocks), NT from the block's
# columns (<= 8: 1, <= 32: 4, else 8)
SK = {"A": (3001, 16, 8, 0),        # fwd NT 1, dX NT 2, dW 2x4
      "B": (2048, 8, 12, 0),        # fwd NT 2, dX NT 1, dW 2x1
      "C": (1500, 20, 30, 0),       # fwd NT 4, dX NT 4, dW 2x4
      "C4": (700, 4, 32, 0),        # fwd NT 4 (K < 8)
      "D": (1200, 40, 6, 0),        # fwd NT 1, dX NT 8, dW 2x8
      "E": (1000, 6, 40, 0),        # fwd NT 8, dX NT 1, dW 4x1
      "F": (2000, 38, 40, 0),       # fwd NT 8, dX NT 8, dW 4x4 + 4x1 (two K blocks)
      "G": (999, 13, 5, 1)}         # misaligned x, K and N not multiples of 4: scalar loads
# wgmma: resident weight (one n tile, <= 4 k blocks), streamed weight (K > 128 or N > 128), odd widths zero-padded by
# ops.linear, the 32-wide layer on the rows kernel, a misaligned x (copied to an aligned buffer by ops)
TC = {"R": (3000, 64, 96, 0), "R8": (1000, 8, 32, 0), "S": (2000, 200, 160, 0), "P": (777, 130, 66, 0),
      "MA": (3000, 128, 128, 1)}
# fused MLP layer (N = 32 out, K = 8 / 16 / 32 / 64 in: mlp_layer_bwd_kernel<NT> from ml_nt); "L64" runs with the
# fused route opened to K = 64
LAYER = {"L8": (3001, 8, 32, 0), "L16": (2000, 16, 32, 0), "L32": (5000, 32, 32, 0), "L32m": (1000, 32, 32, 1),
         "L64": (1500, 64, 32, 0), "W": (3000, 128, 128, 0), "W1": (1000, 128, 96, 1)}


def _gemm_cases():
    cases = []

    def add(kernel, via, *keys, ffma=False):
        table = {"linear": {**SK, **TC}, "layer": LAYER}[via]
        cases.append(dict(kind="gemm", kernel=kernel, via=via, shapes=[table[k] for k in keys], ffma=ffma))
    rm, dm = "skinny_rows_mma_kernel", "skinny_dw_mma_kernel"
    add(kname(rm, True, 1), "linear", "A", "G")
    add(kname(rm, True, 2), "linear", "B")
    add(kname(rm, True, 4), "linear", "C", "C4")
    add(kname(rm, True, 8), "linear", "E", "F")
    add(kname(rm, False, 1), "linear", "B", "E")
    add(kname(rm, False, 2), "linear", "A", "G")
    add(kname(rm, False, 4), "linear", "C")
    add(kname(rm, False, 8), "linear", "D", "F")
    add(kname(dm, 2, 1), "linear", "B")
    add(kname(dm, 2, 4), "linear", "A", "C", "G")
    add(kname(dm, 2, 8), "linear", "D")
    add(kname(dm, 4, 1), "linear", "E")
    add(kname(dm, 4, 4), "linear", "F")
    add("skinny_dw_reduce_cols_kernel", "linear", "A")
    add(kname("tc::tc_rows_kernel", True), "linear", "R", "R8", "MA")
    add(kname("tc::tc_rows_kernel", False), "linear", "S", "P")
    add("tc::tc_dw_kernel", "linear", "R", "MA")
    add("tc::dw_reduce_kernel", "linear", "R")
    add("tc::split_weight_kernel", "linear", "R")
    add("tc::bn_stats_finalize_kernel", "layer", "W", "W1")
    add(kname("mlp_layer_bwd_kernel", 1), "layer", "L8")
    add(kname("mlp_layer_bwd_kernel", 2), "layer", "L16")
    add(kname("mlp_layer_bwd_kernel", 4), "layer", "L32", "L32m")
    add(kname("mlp_layer_bwd_kernel", 8), "layer", "L64")
    add("mlp_dw_reduce_kernel", "layer", "L32")
    # DVA_SKINNY=ffma (read once per process): the fp32-pipe kernels, run in a child process
    for k in (kname("skinny_rows_kernel", True), kname("skinny_rows_kernel", False), "skinny_dw_kernel",
              "skinny_dw_reduce_kernel"):
        cases.append(dict(kind="gemm", kernel=k, via="linear", shapes=[SK["A"], SK["G"], SK["D"]], ffma=True))
    return cases


CASES = _pool_cases() + _bn_cases() + _gemm_cases()
CASE_IDS = [c["kernel"] for c in CASES]


# ------------------------------------------------------------------------------------------------
# pool inputs and references
# ------------------------------------------------------------------------------------------------
POOL_LENGTHS = (0, 1, 2, 31, 32, 33)


def pool_inputs(conf, seed=0):
    """CPU inputs of a pool configuration: map x [B, C, H, W] in the storage type (values repeated across pixels:
    ties), views of POOL_LENGTHS and short random lengths, duplicated pixels inside views, border pixels, for the
    plain gather out-of-range pixels and image ids (clamped by the kernels); interp at 2x - 4x the map size."""
    dt, pix, route, red, interp = conf
    geo = pool_geometry(route, dt)
    B, C, H, W = geo["B"], geo["C"], geo["H"], geo["W"]
    gen = torch.Generator().manual_seed(1000 * seed + 97 * red + 13 * int(interp) + C + H)
    rnd = torch.poisson(torch.full((24,), 2.5), generator=gen).long().tolist()
    counts = torch.tensor(list(POOL_LENGTHS) + rnd)[torch.randperm(len(POOL_LENGTHS) + len(rnd), generator=gen)]
    ptr = ptr_of(counts)
    Vw, P = counts.numel(), int(ptr[-1])
    images = torch.randint(0, B, (Vw,), generator=gen)
    msz = (4 * W - 1, 2 * H + 1) if interp else None
    lim_x, lim_y = (msz if interp else (W, H))
    px = torch.randint(0, lim_x, (P,), generator=gen)
    py = torch.randint(0, lim_y, (P,), generator=gen)
    px[0::9], py[1::9] = 0, lim_y - 1                      # border pixels
    px[2::9], py[3::9] = lim_x - 1, 0
    if not interp:                                       # clamped into the map, like the reference after clamping
        px[4::23], py[5::23], px[6::29] = -3, lim_y + 7, lim_x + 5
        nz = torch.nonzero(counts).view(-1)
        images[nz[0]], images[nz[-1]] = B + 1, -1
    for i in range(Vw):                                  # duplicated pixels: ties between slots of one view
        p0, n = int(ptr[i]), int(counts[i])
        if n >= 2 and i % 3 == 0:
            px[p0 + 1], py[p0 + 1] = px[p0], py[p0]
        if n >= 3 and i % 4 == 1:
            px[p0 + n - 1], py[p0 + n - 1] = px[p0], py[p0]
    pixels = torch.stack([px, py], 1).to(PIX_DT[pix])
    x = torch.randn(B, C, H, W, generator=gen)
    flat = x.view(B, C, H * W)
    flat[:, :, 3::7] = flat[:, :, 3:4]                   # equal values at distinct pixels
    x = x.to(DTYPES[dt])
    gout = torch.randn(Vw, C, generator=gen).to(DTYPES[dt])
    corners = 4 if interp else 1
    if route == "nchw":
        assert P * corners < 0.25 * B * H * W, "must stay below the transposition share"
    if route == "nchw_t":
        assert P * corners >= 0.25 * B * H * W
    return dict(conf=conf, dtype=dt, red=RED_NAMES[red], interp=interp, x=x, images=images, pixels=pixels,
                ptr=ptr, counts=counts, msz=msz, gout=gout, off=geo["off"], cl=geo["cl"])


def _clamped(inp):
    B, C, H, W = inp["x"].shape
    view = O.dense_index(inp["ptr"])
    b = inp["images"].clamp(0, B - 1)
    pix = inp["pixels"].long()
    if inp["msz"] is None:
        pix = torch.stack([pix[:, 0].clamp(0, W - 1), pix[:, 1].clamp(0, H - 1)], 1)
    return b, b[view], pix, view


def pool_values(inp, x=None):
    """[P, C] fp32 values the kernels pool (exact float64 copies of fp32 numbers)."""
    x = (inp["x"] if x is None else x).float()
    b, b_slot, pix, _ = _clamped(inp)
    if inp["msz"] is None:
        return O.feature_map_gather(x, b, pix, inp["ptr"]).double()
    return torch.from_numpy(IO.sparse_interpolation_pixels(x.numpy(), pix.numpy(), b_slot.numpy(),
                                                           inp["msz"])).double()


def pool_forward_ref(inp, vals=None, ptr=None, arg_fn=DO.first_arg):
    """(reference, bound or None for bit-equality, arg) of the forward."""
    vals = pool_values(inp) if vals is None else vals
    ptr = inp["ptr"] if ptr is None else ptr
    dt, red = inp["dtype"], inp["red"]
    n = (ptr[1:] - ptr[:-1]).double().view(-1, 1)
    if red in ("max", "min"):
        arg = torch.from_numpy(arg_fn(vals.float().numpy(), ptr.numpy(), red))
        ref = torch.where(arg >= 0, vals.gather(0, arg.clamp(min=0) - int(ptr[0])), torch.zeros_like(vals[:1]))
        return round_to(ref, dt), None, arg
    ref = S_segment_csr(vals, ptr, reduce="sum")
    acc = KE * n * S_segment_csr(vals.abs(), ptr, reduce="sum")
    if red == "mean":
        ref, acc = ref / n.clamp(min=1), acc / n.clamp(min=1)
    return ref, U_S[dt] * ref.abs() + acc + TINY[dt], None


def pool_contributions(inp, arg, last=False):
    """(keys [S], values [S, C] exact fp32) of the map-gradient scatter: key = (b H + y) W + x of the map pixel."""
    B, C, H, W = inp["x"].shape
    b, b_slot, pix, view = _clamped(inp)
    ptr, counts = inp["ptr"], inp["counts"]
    n = counts[view]
    val = inp["gout"].float()[view]
    if inp["red"] == "mean":
        val = val / n.float().view(-1, 1)
    if inp["red"] in ("max", "min"):
        slot = torch.arange(int(ptr[0]), int(ptr[-1])).view(-1, 1)
        on = (n.view(-1, 1) == 1) | (arg[view] == slot)
        val = torch.where(on, val, torch.zeros_like(val))
    if inp["msz"] is None:
        return (b_slot * H + pix[:, 1]) * W + pix[:, 0], val
    (top, bottom, left, right), wts = DO.bilinear_footprint(pix.numpy(), inp["msz"], H, W)
    rows = [torch.from_numpy(r.astype(np.int64) - 1).clamp(0, H - 1) for r in (top, bottom)]
    cols = [torch.from_numpy(c.astype(np.int64) - 1).clamp(0, W - 1) for c in (left, right)]
    corner = [(rows[0], cols[0]), (rows[0], cols[1]), (rows[1], cols[0]), (rows[1], cols[1])]
    keys = torch.stack([(b_slot * H + r) * W + c for r, c in corner], 1).reshape(-1)
    vals = torch.stack([torch.from_numpy(wk).view(-1, 1) * val for wk in wts], 1).reshape(-1, C)
    return keys, vals


def pool_backward_ref(inp, arg, contrib=None):
    """(reference [B, H, W, C] float64, bound) of the atomic map gradient."""
    B, C, H, W = inp["x"].shape
    keys, vals = pool_contributions(inp, arg) if contrib is None else contrib
    vals = vals.double()
    ref = torch.zeros(B * H * W, C, dtype=torch.float64).index_add_(0, keys, vals)
    absum = torch.zeros(B * H * W, C, dtype=torch.float64).index_add_(0, keys, vals.abs())
    cnt = torch.bincount(keys, minlength=B * H * W).double().view(-1, 1)
    dt = inp["dtype"]
    bound = KE * (cnt + 1) * absum + U_S[dt] * ref.abs() + TINY[dt]
    return ref.view(B, H, W, C), bound.view(B, H, W, C)


def pool_det_ref(inp, arg):
    """Deterministic map gradient [B, H, W, C] float64: map_grad_ordered rounded to the storage type."""
    B, C, H, W = inp["x"].shape
    g = DO.map_grad_ordered((B, H, W, C), inp["gout"].float().numpy(), inp["images"].numpy(),
                            inp["pixels"].long().numpy(), inp["ptr"].numpy(), inp["red"],
                            None if arg is None else arg.numpy(), inp["msz"])
    return round_to(torch.from_numpy(g).double(), inp["dtype"])


def last_arg(vals, aptr, reduce):
    """first_arg with ties won by the last slot (an injected bug)."""
    aptr = np.asarray(aptr)
    P = int(aptr[-1]) - int(aptr[0])
    rev = np.asarray(vals)[::-1]
    counts = aptr[1:] - aptr[:-1]
    rptr = np.concatenate([[0], np.cumsum(counts[::-1])])
    a = DO.first_arg(rev, rptr, reduce)[::-1]
    return np.where(a >= 0, P - 1 - a + int(aptr[0]), -1)


# ------------------------------------------------------------------------------------------------
# BatchNorm reference and bounds
# ------------------------------------------------------------------------------------------------
def bn_inputs(dt, cfg, seed=0):
    gen = torch.Generator().manual_seed(1000 * seed + cfg["R"] + 7 * cfg["C"] + int(cfg["training"]))
    R, C = cfg["R"], cfg["C"]
    z = torch.randn(R, C, generator=gen) * 2 + 0.5
    if cfg["special"]:
        z[:, 0] = 1.25                                   # constant column: var = 0, invstd = 1 / sqrt(eps)
        if C > 1:
            z[:, 1] = 1000.0 + torch.randn(R, generator=gen)   # |mean| / std = 1e3: the row-0 shift matters
    gamma = (torch.rand(C, generator=gen) + 0.5) if cfg["affine"] else None
    beta = (torch.randn(C, generator=gen) * 0.3) if cfg["affine"] else None
    rm = torch.randn(C, generator=gen)
    rv = torch.rand(C, generator=gen) + 0.5
    if cfg["special"] and not cfg["training"]:
        rm[0], rv[0] = 1.25, 0.0
    dy = torch.randn(R, C, generator=gen).to(DTYPES[dt])
    return dict(z=z.to(DTYPES[dt]), gamma=gamma, beta=beta, rm=rm, rv=rv, dy=dy, eps=1e-5,
                momentum=cfg["momentum"], tracked=3, training=cfg["training"], dtype=dt, vec=None)


def bn_chain_length(R, C, vec):
    G = min(-(-R // 64), 4 * NUM_SMS) if R > 0 else 1
    RG = 256 // min(C // vec if vec > 1 else C, 256)
    return -(-(-(-R // G)) // RG) + RG + 2


def epilogue_stats_error(z):
    """(dS, dQ) [C]: error bounds of the column sums S = sum z and Q = sum z^2 that bn_stats_finalize_kernel
    rebuilds from the wgmma rows kernel's epilogue (module docstring), on exact z."""
    R, C = z.shape
    m_tiles = -(-R // 128)
    ctas = min(m_tiles, NUM_SMS)
    cta = (torch.arange(R) // 128) % ctas                # tiles b, b + ctas, ... go to CTA b
    sh = z[128 * torch.arange(ctas)]                     # row 0 of each CTA's first tile
    d = z - sh[cta]
    s = torch.zeros(ctas, C, dtype=torch.float64).index_add_(0, cta, d)
    q = torch.zeros(ctas, C, dtype=torch.float64).index_add_(0, cta, d * d)
    S1 = torch.zeros(ctas, C, dtype=torch.float64).index_add_(0, cta, d.abs())
    ds = KE * 17 * S1 + U32 * s.abs()
    dq = KE * 17 * q + U32 * q
    return ds.sum(0), (dq + 2 * sh.abs() * ds).sum(0)


def bn_reference(inp, vec, dzin=None, epilogue=False, unbiased_norm=False, slope_pos=False, unshifted_f32=False):
    """Float64 BatchNorm + LeakyReLU(0.2) forward / backward on the stored z, with the bounds of the module
    docstring.  dzin: per-element error of z (GEMM output).  epilogue: the batch statistics come from the wgmma
    rows kernel's epilogue (ops.linear_bn_act) instead of bn_stats_kernel.  The remaining flags inject bugs."""
    z = inp["z"].double()
    R, C = z.shape
    dt, eps, training = inp["dtype"], inp["eps"], inp["training"]
    gamma = inp["gamma"].double() if inp["gamma"] is not None else torch.ones(C, dtype=torch.float64)
    beta = inp["beta"].double() if inp["beta"] is not None else torch.zeros(C, dtype=torch.float64)
    dzin = torch.zeros_like(z) if dzin is None else dzin
    m = inp["momentum"] if inp["momentum"] is not None else 1.0 / (inp["tracked"] + 1)
    L = bn_chain_length(R, C, vec)
    if training:
        mu = z.mean(0)
        var = ((z - mu) ** 2).mean(0)
        if unshifted_f32:                               # plain fp32 sums of z and z^2, sequential
            z32 = inp["z"].float().numpy()
            s = np.cumsum(z32, 0, dtype=np.float32)[-1]
            q = np.cumsum(z32 * z32, 0, dtype=np.float32)[-1]
            ms = s / np.float32(R)
            var = torch.from_numpy(np.maximum(q / np.float32(R) - ms * ms, 0).astype(np.float64))
        if epilogue:
            dS, dQ = epilogue_stats_error(z)
            dmu = dS / R + KE * mu.abs() + dzin.mean(0)
            dvar = dQ / R + 2 * mu.abs() * dS / R + 2.0 ** -50 * (z * z).mean(0) + 2 * ((z - mu).abs() * dzin).mean(0)
        else:
            d = z - z[0]
            S1, S2 = d.abs().sum(0), (d * d).sum(0)
            dmu = KE * (L * S1 / R + mu.abs()) + dzin.mean(0)
            dvar = KE * L * (S2 + 2 * (mu - z[0]).abs() * S1) / R + 2 * ((z - mu).abs() * dzin).mean(0)
        nvar = var * R / (R - 1) if (unbiased_norm and R > 1) else var
        inv = 1 / torch.sqrt(nvar + eps)
        dinv = inv * (dvar / (2 * (var + eps)) + KE)
    else:
        mu, var = inp["rm"].double(), inp["rv"].double()
        inv = 1 / torch.sqrt(var + eps)
        dmu, dvar, dinv = torch.zeros(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64), KE * inv
    zh = (z - mu) * inv
    a = gamma * zh + beta
    da = gamma.abs() * (inv * (dmu + dzin) + (z - mu).abs() * dinv) + \
        KE * (gamma.abs() * inv * (z.abs() + mu.abs()) + beta.abs())
    pos = (a > 0) if not slope_pos else (a <= 0)
    y = torch.where(pos, a, SLOPE * a)
    flip = a.abs() <= da
    us, tiny = U_S[dt], TINY[dt]
    b_y = da + us * y.abs() + tiny + flip.double() * (1 - SLOPE) * a.abs()
    dy = inp["dy"].double()
    g = torch.where(pos, dy, SLOPE * dy)
    F0 = (flip.double() * (1 - SLOPE) * dy.abs()).sum(0)
    F1 = (flip.double() * (1 - SLOPE) * (dy * zh).abs()).sum(0)
    dzh = inv * (dmu + dzin) + (z - mu).abs() * dinv + KE * zh.abs()
    dbeta, dgamma = g.sum(0), (g * zh).sum(0)
    b_dbeta = KE * L * g.abs().sum(0) + F0 + 2.0 ** -126
    b_dgamma = KE * L * (g * zh).abs().sum(0) + (g.abs() * dzh).sum(0) + F1 + 2.0 ** -126
    sc = gamma * inv
    dsc = gamma.abs() * dinv + KE * sc.abs()
    k0, k1 = (dbeta / R, dgamma / R) if training else (torch.zeros(C, dtype=torch.float64),) * 2
    dk0, dk1 = (b_dbeta / R, b_dgamma / R) if training else (torch.zeros(C, dtype=torch.float64),) * 2
    q = g - k0 - zh * k1
    dz = sc * q
    b_dz = dsc * q.abs() + sc.abs() * (flip.double() * (1 - SLOPE) * dy.abs() + dk0 + zh.abs() * dk1
                                       + k1.abs() * dzh + KE * (g.abs() + k0.abs() + (zh * k1).abs())) \
        + us * dz.abs() + tiny
    res = dict(y=y, b_y=b_y, dz=dz, b_dz=b_dz, dgamma=dgamma, b_dgamma=b_dgamma, dbeta=dbeta, b_dbeta=b_dbeta,
               mu=mu, dmu=dmu, inv=inv, dinv=dinv, a=a, flip=flip)
    if training:
        unb = var * R / (R - 1) if R > 1 else var
        rm = (1 - m) * inp["rm"].double() + m * mu
        rv = (1 - m) * inp["rv"].double() + m * unb
        res.update(rm=rm, b_rm=m * dmu + KE * rm.abs() + 2.0 ** -126,
                   rv=rv, b_rv=m * dvar * (R / (R - 1) if R > 1 else 1.0) + KE * rv.abs() + 2.0 ** -126)
    return res


# ------------------------------------------------------------------------------------------------
# GEMM bounds
# ------------------------------------------------------------------------------------------------
def dw_chain(family, M, N, K):
    """Longest fp32 chain of a dW element: rows one CTA accumulates + the CTA partials summed after it, from the
    launch's grid (skinny_dw_mma: grid_cap(M, 64, 4); skinny_dw: grid_cap(M, 128, 3); mlp: grid_cap(M, 64, 2 or 3);
    tc_dw: 32-row blocks split over 132 / (n tiles * k tiles) CTAs per output tile)."""
    def per_cta(tile, cap):
        tiles = -(-M // tile)
        P = min(tiles, cap)
        return -(-tiles // P) * tile + P
    if family == "mma":
        return per_cta(64, 4 * NUM_SMS)
    if family == "ffma":
        return per_cta(128, 3 * NUM_SMS)
    if family == "mlp":
        nt = 1 if K <= 8 else 2 if K <= 16 else 4 if K <= 32 else 8
        return per_cta(64, (2 if nt == 8 else 3) * NUM_SMS)
    blocks = -(-M // 32)
    sp = min(max(NUM_SMS // (-(-N // 128) * -(-K // 128)), 1), blocks)
    return -(-blocks // sp) * 32 + sp


def gemm_bound(absprod, L, extra=0.0):
    """(ke (L + 2) + 2^-20) sum |a b| + tiny (+ the propagated error of an inexact operand)."""
    return (KE * (L + 2) + 2.0 ** -20) * absprod + extra + 2.0 ** -126


def tf32(t):
    """Round fp32 values to TF32 (10 explicit mantissa bits), to nearest."""
    b = t.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32).double()


# ------------------------------------------------------------------------------------------------
# CPU tests
# ------------------------------------------------------------------------------------------------
def test_case_table_matches_library():
    path = _lib_path()
    if not os.path.exists(path):
        pytest.fail(f"{path} is not built")
    assert len(CASE_IDS) == len(set(CASE_IDS)), "one case per instantiation"
    built = library_kernels(path, FAMILIES)
    table = set(CASE_IDS)
    assert built == table, {"compiled without a case": sorted(built - table),
                            "case without an instantiation": sorted(table - built)}
    fam = [parse_kernel("dva::" + k)[0] for k in table]
    counts = {f: fam.count(f) for f in set(fam)}
    assert counts["gather_pool_fwd_cl_kernel"] == 192 and counts["det::gather_pool_bwd_det_cl_kernel"] == 96
    assert counts["gather_pool_fwd_kernel"] == 96 and counts["det::gather_pool_bwd_det_kernel"] == 48
    assert sum(counts[f] for f in ("bn_stats_kernel", "bn_apply_kernel", "bn_bwd_reduce_kernel",
                                   "bn_bwd_apply_kernel")) == 24


def test_parse_nested_namespaces():
    assert parse_kernel("void dva::det::gather_pool_bwd_det_cl_kernel<__half, 16, 0, true>(__half const*, long)") == \
        ("det::gather_pool_bwd_det_cl_kernel", ("__half", "16", "0", "true"))
    assert canonical("void dva::tc::tc_rows_kernel<true>(CUtensorMap, CUtensorMap, CUtensorMap, dva::tc::RowsParams)") \
        == "tc::tc_rows_kernel<true>"
    assert canonical("dva::tc::dw_reduce_kernel(float const*, float*, int, int, int, int, int, long)") == \
        "tc::dw_reduce_kernel"
    assert canonical("void dva::bk::count_keys<1, dva::det::PixelKey<int, false>>(long)") is None


def test_every_pool_configuration_routes_as_intended():
    """The inputs of each route satisfy the host dispatch's conditions (gp_cl_vec_ok, with_lpr, the NCHW
    transposition share of _GatherPool.forward)."""
    for conf in POOL_CONFS[::7] + POOL_CONFS[-9:]:
        dt, pix, route, red, interp = conf
        geo = pool_geometry(route, dt)
        V, C = V16[dt], geo["C"]
        if route.startswith("lpr") or route == "nchw_t":
            cv = C // V
            assert C % V == 0 and C % 4 == 0
            lpr = 4 if cv <= 4 else 8 if cv <= 8 else 16 if cv <= 16 else 32
            assert lpr == (16 if route == "nchw_t" else int(route[3:]))
        elif route == "cl_scalar":
            assert C % V != 0
        pool_inputs(conf)                                # asserts the transposition share


def _buggy_bilinear(inp):
    """Interp values with the top-left and top-right corner weights swapped."""
    x = inp["x"].float().numpy()
    B, C, H, W = x.shape
    b, b_slot, pix, _ = _clamped(inp)
    (top, bottom, left, right), (w00, w01, w10, w11) = DO.bilinear_footprint(pix.numpy(), inp["msz"], H, W)
    pad = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)), mode="edge")
    bb = b_slot.numpy()

    def at(r, c):
        return pad[bb, :, r.astype(np.int64), c.astype(np.int64)].astype(np.float64)
    return torch.from_numpy(w01[:, None] * at(top, left) + w00[:, None] * at(top, right)
                            + w10[:, None] * at(bottom, left) + w11[:, None] * at(bottom, right))


@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
def test_bounds_reject_buggy_pools(dt):
    rejected = {}
    V = V16[dt]
    for interp in (False, True):
        conf_s = (dt, "i32", "lpr8", 0, interp)
        inp = pool_inputs(conf_s, seed=3)
        ref, bnd, _ = pool_forward_ref(inp)
        assert violations(round_to(ref, dt), ref, bnd)[0] == 0
        vals = pool_values(inp)
        ptr, counts = inp["ptr"], inp["counts"]
        keep = torch.ones(int(ptr[-1]), dtype=torch.bool)
        keep[(ptr[1:] - 1)[counts > 0]] = False
        r1, _, _ = pool_forward_ref(inp, vals=vals[keep], ptr=ptr_of(torch.clamp(counts - 1, min=0)))
        rejected[f"drop last pixel interp={interp}"] = violations(round_to(r1, dt), ref, bnd)[0]
        v2 = vals.clone()
        v2[:, V:2 * V] = vals[:, V + 1:2 * V + 1]
        rejected[f"chunk one channel late interp={interp}"] = \
            violations(round_to(pool_forward_ref(inp, vals=v2)[0], dt), ref, bnd)[0]
        if interp:
            rejected["bilinear corner weights swapped"] = \
                violations(round_to(pool_forward_ref(inp, vals=_buggy_bilinear(inp))[0], dt), ref, bnd)[0]
        if dt != "f32":
            rejected[f"round toward zero interp={interp}"] = \
                violations(round_to(ref, dt, toward_zero=True), ref, bnd)[0]
        inp_m = pool_inputs((dt, "i32", "lpr8", 1, interp), seed=3)
        ref_m, bnd_m, _ = pool_forward_ref(inp_m)
        n = inp_m["counts"].double().view(-1, 1)
        rejected[f"mean over n - 1 interp={interp}"] = \
            violations(round_to(ref_m * n / (n - 1).clamp(min=1), dt), ref_m, bnd_m)[0]
        if interp:      # bilinear samples of distinct pixels rarely tie; duplicated pixels send ties to one place
            continue
        # ties won by the last slot: the forward value is the same, the gradient lands on another pixel
        inp_x = pool_inputs((dt, "i32", "lpr8", 2, interp), seed=3)
        _, _, arg = pool_forward_ref(inp_x)
        gref, gbnd = pool_backward_ref(inp_x, arg)
        assert violations(gref, gref, gbnd)[0] == 0
        _, _, arg_l = pool_forward_ref(inp_x, arg_fn=last_arg)
        assert not torch.equal(arg, arg_l), "the inputs must hold ties"
        gl, _ = pool_backward_ref(inp_x, arg_l)
        rejected[f"ties to the last pixel interp={interp}"] = violations(round_to(gl, dt), gref, gbnd)[0]
        assert not torch.equal(pool_det_ref(inp_x, arg), pool_det_ref(inp_x, arg_l))
    assert all(v > 0 for v in rejected.values()), rejected


def test_bounds_reject_buggy_batchnorm():
    rejected = {}
    cfg = dict(R=1000, C=16, training=True, affine=True, momentum=0.1, z_off=0, special=True)
    inp = bn_inputs("f32", cfg, seed=5)
    ref = bn_reference(inp, 4)
    for k in ("y", "dz", "dgamma", "dbeta", "rm", "rv"):
        assert violations(ref[k].float().double(), ref[k], ref["b_" + k])[0] == 0, k
    rejected["unbiased variance in the normalisation"] = \
        violations(bn_reference(inp, 4, unbiased_norm=True)["y"], ref["y"], ref["b_y"])[0]
    rejected["d gamma and d beta swapped"] = violations(ref["dbeta"], ref["dgamma"], ref["b_dgamma"])[0]
    rejected["slope on the positive side"] = \
        violations(bn_reference(inp, 4, slope_pos=True)["y"], ref["y"], ref["b_y"])[0]
    bad = bn_reference(inp, 4, unshifted_f32=True)
    rejected["unshifted fp32 statistics"] = violations(bad["y"][:, 1], ref["y"][:, 1], ref["b_y"][:, 1])[0]
    assert all(v > 0 for v in rejected.values()), rejected


@pytest.mark.parametrize("M,K,N", [(2000, 16, 8), (1000, 32, 32), (500, 40, 12)])
def test_bounds_reject_buggy_gemms(M, K, N):
    gen = torch.Generator().manual_seed(M + K + N)
    x = torch.randn(M, K, generator=gen)
    w = torch.randn(N, K, generator=gen) / math.sqrt(K)
    x64, w64 = x.double(), w.double()
    ref = x64 @ w64.t()
    bnd = gemm_bound(x64.abs() @ w64.abs().t(), K)
    assert violations(ref.float().double(), ref, bnd)[0] == 0
    rejected = {"1xTF32": violations(tf32(x) @ tf32(w).t(), ref, bnd)[0]}
    if K > 32:
        rejected["last K block dropped"] = violations(x64[:, :32] @ w64[:, :32].t(), ref, bnd)[0]
    xh, wh = tf32(x), tf32(w)
    xl, wl = tf32(x64 - xh), tf32(w64 - wh)
    rejected["lo hi correction dropped"] = violations(xh @ wh.t() + xh @ wl.t(), ref, bnd)[0]
    assert violations(xh @ wh.t() + xh @ wl.t() + xl @ wh.t(), ref, bnd)[0] == 0, "3xTF32 itself must pass"
    assert all(v > 0 for v in rejected.values()), rejected


def test_dw_bound_reach():
    """What the bound does and does not separate on a dW chain (L = rows per CTA + CTA partials, here
    skinny_dw_mma's 64 + 47 for M = 3000).  A dropped 64-row tile, or one CTA's partial summed twice, is rejected.
    1xTF32 is not: over a long chain ke (L + 2) sum |a b| is ~2^-14 of sum |a b|, far above the random 1xTF32 error
    of the sum (~sqrt(M) 2^-12 |a b|).  1xTF32 is rejected on the rows kernels' chains (L = K <= 40), see
    test_bounds_reject_buggy_gemms."""
    M, N, K = 3000, 8, 16
    gen = torch.Generator().manual_seed(11)
    g, x = torch.randn(M, N, generator=gen), torch.randn(M, K, generator=gen)
    g64, x64 = g.double(), x.double()
    ref = g64.t() @ x64
    L = dw_chain("mma", M, N, K)
    assert L == 64 + 47
    bnd = gemm_bound(g64.abs().t() @ x64.abs(), L)
    assert violations(ref.float().double(), ref, bnd)[0] == 0
    assert violations(g64[64:].t() @ x64[64:], ref, bnd)[0] > 0, "a dropped row tile"
    assert violations(ref + g64[:64].t() @ x64[:64], ref, bnd)[0] > 0, "one partial summed twice"
    assert violations(tf32(g).t() @ tf32(x), ref, bnd)[0] == 0, "1xTF32 lies inside the dW bound"
