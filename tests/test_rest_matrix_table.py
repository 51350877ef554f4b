"""Kernel matrix of every kernel outside the view-attention / segment / qk table (tests/test_kernel_matrix_table.py)
and the pool / BatchNorm / GEMM table (tests/test_pool_gemm_matrix_table.py): the grid k-NN and the neighbourhood
features (knn_features.cu), the native mapping build (mapping_build.cu), the bucket index (bucket_sort.cuh) and its
users, the deterministic row scatter (segment_csr.cu), the projection / splat / z-buffer kernels (zbuffer.cu), the
CSR bookkeeping (csr_build.cu), the CSR log-softmax NLL (csr_nll.cu) and the image kernels (image_transforms.cu,
image_resample.cu, image_color.cu).

tests/test_gpu_rest_matrix.py runs every case on the GPU under the kernel recorder and asserts, by name, the kernels
the case must launch.  This file checks, without a GPU, that
  * the case table holds exactly the kernels of these families compiled into libdva_b200.so;
  * the three tables together hold every dva:: kernel of the library, with no family filter: a new kernel anywhere
    fails here.  The bucket-index kernels bk::scan_block_sums / scan_of_sums / scan_apply / order_by_id are static
    in a header, so each translation unit that includes it compiles its own copy under the same name; the table
    holds each name once and lists every user, and every user gets its own GPU case;
  * every bound can fail: plausible bugs injected into the references break them.

References and bounds (u32 = 2^-24, u_s = half an ulp of the storage type, ke = 8 u32):
  k-NN (self and query / search, k <= 64 and <= 128)   the fp32 brute force with the kernel's arithmetic
        ((dx*dx + dy*dy) + dz*dz, no contraction) and its (d2, index) order: indices and d2 bit-equal.
  neighbourhood features   the fp32 restatement (oracle/neighborhood_oracle.py): bit-equal, inf and NaN included.
  mapping build, view_cat_sorting, CSR bookkeeping   numpy stable lexsort (oracle/visibility_oracle.py), independent
        of the torch host path: every integer bit-equal; view feature means within
        2 u32 |ref| + 8 u32 (n - 1) sum|f| / n (the kernel sums the n items of a view in order in fp32, then
        multiplies by a rounded reciprocal).
  bucket-index users   the deterministic pool and row-scatter gradients bit-equal to oracle/deterministic_oracle.py;
        PickImagesFromMemoryCredit equal to its fixture; the coverage index equal to the CPU path.
  scatter_add_rows_det   the ordered fp32 sum (ascending source row) bit-equal; heuristic_arg bit-equal (the picked
        rows); gate_reduce under the view-attention gate-gradient bound of test_kernel_matrix_table.py.
  projection, splat boxes, z-buffer   the C oracle (oracle/visibility_oracle.c): bit-equal, ties to the lower index.
  NLL   float64 log_softmax + nll_loss (mean).  mag_v = max_j |x_vj| + |lse_v| (float64), over the counted rows:
        loss   |got - ref| <= ke (K + 2) mean(mag_v) + u32 |ref|
        grad   u_s |ref| + ke ((K + 2) mag_v p_vj + 1) |g| / count + tiny   (p = float64 softmax, g = grad of loss)
  resample, nonstatic mask, to_float, jitter   oracle/image_resample_oracle.py and oracle/color_oracle.py: bit-equal.
"""
import os

import numpy as np
import pytest
import torch

from test_kernel_matrix_table import (CPP, DTYPES, K_ERR, TINY, U32, U_S, _lib_path, kname, library_kernels,
                                      parse_kernel, violations)
import test_kernel_matrix_table as KM
import test_pool_gemm_matrix_table as PG

KE = K_ERR * U32
FAMILIES = ("knn_grid_kernel", "knn_cell_ids_kernel", "neighborhood_features_kernel",
            "mb::order_points", "mb::emit_points", "mb::finish_counts", "mb::view_cat_sorting_kernel",
            "bk::scan_block_sums", "bk::scan_of_sums", "bk::scan_apply", "bk::order_by_id", "bk::count_keys",
            "bk::scatter_keys", "scatter_add_rows_det_kernel", "heuristic_arg_kernel", "gate_reduce_kernel",
            "project_camera_kernel", "project_equirect_kernel", "splat_boxes_kernel", "splat_boxes_width_kernel",
            "fill_u64_kernel", "zbuffer_raster_kernel", "zbuffer_resolve_kernel", "zbuffer_centres_kernel",
            "csr_pointers_kernel", "csr_select_values_kernel", "csr_nll_fwd_kernel", "csr_nll_bwd_kernel",
            "csr_nll_finalize_kernel", "stats_accumulate", "stats_init", "stats_finalize", "center_roll_kernel",
            "remap_kernel", "coverage_fill", "coverage_pick_kernel", "resample_h_kernel", "resample_v_kernel",
            "nonstatic_mask_kernel", "to_float_kernel", "to_float_vec_kernel", "jitter_sum_kernel",
            "jitter_apply_kernel")
SCAN_CARRY_BUCKETS = 1024 * 2048        # more buckets than this: bk::scan_of_sums carries across passes
PIXELS = {"i16": "short", "i32": "int", "i64": "long"}


def canonical(name):
    return KM.canonical(name, FAMILIES)


# ------------------------------------------------------------------------------------------------
# the case table: kernel -> the scenarios of tests/test_gpu_rest_matrix.py that must launch it
# ------------------------------------------------------------------------------------------------
def _key(functor, nk=1):
    return f"{nk}, dva::{functor}"


# the users of the bucket index, each with a case above SCAN_CARRY_BUCKETS buckets
BK_USERS = {"mapping": ("mapping_i16", "mapping_big"),
            "det_pool": ("det_pool", "det_pool_big"),
            "det_rows": ("det_rows_f32", "det_rows_big"),
            "coverage": ("coverage", "coverage_big")}


def _cases():
    c = {}

    def add(kernel, *scenarios):
        assert kernel not in c, kernel
        c[kernel] = list(scenarios)

    for kmax in (64, 128):
        for coarse in (False, True):
            add(kname("knn_grid_kernel", kmax, coarse), f"knn_{'query' if coarse else 'self'}{kmax}")
    add("knn_cell_ids_kernel", "knn_self64", "knn_query64")
    add("neighborhood_features_kernel", "nbr_features")
    for px, T in PIXELS.items():
        add(kname("mb::order_points", T), f"mapping_{px}")
        add(kname("mb::emit_points", T), f"mapping_{px}")
    add("mb::finish_counts", "mapping_i16", "mapping_big")
    add("mb::view_cat_sorting_kernel", "view_cat")
    # bucket index: the scans in every user, the ordering pass in the users that order their buckets
    for k in ("bk::scan_block_sums", "bk::scan_of_sums", "bk::scan_apply"):
        add(k, *[s for u in BK_USERS.values() for s in u])
    add("bk::order_by_id", *BK_USERS["det_pool"], *BK_USERS["det_rows"])
    keys = {_key("mb::PointKey"): BK_USERS["mapping"], _key("RowKey"): BK_USERS["det_rows"],
            _key("KeyFrom"): BK_USERS["coverage"]}
    for px in ("short", "int"):
        keys[_key(f"det::PixelKey<{px}, false", 1)] = ("det_pool",) + (("det_pool_big",) if px == "int" else ())
        keys[_key(f"det::PixelKey<{px}, true", 4)] = ("det_pool",)
    for kk, scen in keys.items():
        add(f"bk::count_keys<{kk}>", *scen)
        add(f"bk::scatter_keys<{kk}>", *scen)
    for dt in DTYPES:
        for vec in (KM.V16[dt] if dt != "f32" else 4, 1):
            add(kname("scatter_add_rows_det_kernel", CPP[dt], vec), f"det_rows_{dt}")
    add("heuristic_arg_kernel", "heuristic_arg")
    add("gate_reduce_kernel", "gate_reduce")
    add("project_equirect_kernel", "zbuffer_equirect")
    add("project_camera_kernel", "zbuffer_camera")
    add("splat_boxes_kernel", "zbuffer_equirect", "zbuffer_random")
    add("splat_boxes_width_kernel", "zbuffer_camera")
    for k in ("fill_u64_kernel", "zbuffer_raster_kernel", "zbuffer_resolve_kernel", "zbuffer_centres_kernel"):
        add(k, "zbuffer_equirect", "zbuffer_random")
    add("csr_pointers_kernel", "csr_build")
    add("csr_select_values_kernel", "csr_build")
    for dt in DTYPES:
        add(kname("csr_nll_fwd_kernel", CPP[dt]), f"nll_{dt}")
        add(kname("csr_nll_bwd_kernel", CPP[dt]), f"nll_{dt}")
    add("csr_nll_finalize_kernel", "nll_f32", "nll_edges")
    for px, T in PIXELS.items():
        add(kname("stats_accumulate", T), f"image_stats_{px}")
    add("stats_init", "image_stats_i16")
    add("stats_finalize", "image_stats_i16")
    add("center_roll_kernel", "center_roll")
    add("remap_kernel", "remap")
    add("coverage_fill", "coverage", "coverage_big")
    add("coverage_pick_kernel", "coverage", "coverage_big")
    for C in (1, 2, 3, 4):
        add(kname("resample_h_kernel", C), f"resample_C{C}")
        add(kname("resample_v_kernel", C), f"resample_C{C}")
        add(kname("nonstatic_mask_kernel", C), f"nonstatic_C{C}")
    for T, tag in (("unsigned char", "u8"), ("float", "f32")):
        add(kname("to_float_vec_kernel", T), f"to_float_{tag}_vec")
        add(kname("to_float_kernel", T), f"to_float_{tag}_scalar")
    add("jitter_sum_kernel", "jitter")
    add("jitter_apply_kernel", "jitter")
    return c


TABLE = _cases()
# one GPU case per (kernel, scenario)
CASES = [dict(kernel=k, scenario=s) for k, ss in TABLE.items() for s in ss]
CASE_IDS = [f"{c['kernel']}@{c['scenario']}" for c in CASES]
SCENARIOS = sorted({c["scenario"] for c in CASES})


def all_library_kernels(lib_path):
    """Canonical names of every dva:: kernel compiled into `lib_path`, no family filter."""
    class _All:
        def __contains__(self, _):
            return True
    return library_kernels(lib_path, _All())


# ------------------------------------------------------------------------------------------------
# references shared with the GPU file
# ------------------------------------------------------------------------------------------------
def nll_reference(logits, labels, csr, ignore_index=-1):
    """float64 log_softmax + nll_loss (mean) and its gradient; the per-row magnitude mag_v; count."""
    x = logits.detach().double().cpu().requires_grad_(True)
    lab = labels.cpu()
    target = lab if csr is None else torch.repeat_interleave(lab, (csr[1:] - csr[:-1]).cpu())
    logp = torch.log_softmax(x, -1)
    loss = torch.nn.functional.nll_loss(logp, target, ignore_index=ignore_index)
    g, = torch.autograd.grad(loss, x) if x.shape[0] else (torch.zeros_like(x),)
    xd = x.detach()
    lse = torch.logsumexp(xd, -1) if xd.shape[0] else torch.zeros(0, dtype=torch.float64)
    fin = torch.where(torch.isfinite(xd), xd.abs(), torch.zeros_like(xd))
    mag = (fin.max(-1).values if xd.shape[1] else torch.zeros(xd.shape[0], dtype=torch.float64)) + \
        torch.where(torch.isfinite(lse), lse.abs(), torch.zeros_like(lse))
    counted = target != ignore_index
    return dict(loss=loss.detach(), grad=g, mag=mag, p=torch.softmax(xd, -1), counted=counted,
                count=int(counted.sum()), target=target)


def nll_bounds(ref, K, dt, grad_loss=1.0):
    cnt = max(ref["count"], 1)
    mag = ref["mag"][ref["counted"]]
    b_loss = KE * (K + 2) * (float(mag.mean()) if mag.numel() else 0.0) + U32 * abs(float(ref["loss"]))
    gs = abs(grad_loss) / cnt
    b_grad = U_S[dt] * ref["grad"].abs() + KE * ((K + 2) * ref["mag"].view(-1, 1) * ref["p"] + 1) * gs + TINY[dt]
    return b_loss, b_grad


def mapping_feature_bound(feat, atomic_ptr, ref):
    """2 u32 |ref| + 8 u32 (n - 1) sum|f| / n per view."""
    f = np.abs(np.asarray(feat, dtype=np.float64))
    ap = np.asarray(atomic_ptr)
    n = np.maximum(np.diff(ap), 1)[:, None]
    s = np.add.reduceat(f, ap[:-1], axis=0) if f.shape[0] else np.zeros((0, f.shape[1]))
    return 2 * U32 * np.abs(ref) + K_ERR * U32 * (n - 1) * s / n


def scan_exclusive(counts, drop_carry=False, items=2048, per_pass=1024):
    """Restatement of bk::exclusive_scan: per-block sums, a scan of the block sums in passes of `per_pass`
    blocks (drop_carry: the carry between passes lost), then the in-block prefix; out has n + 1 entries."""
    c = np.asarray(counts, dtype=np.int64)
    nb = (c.size + items - 1) // items
    sums = np.add.reduceat(c, np.arange(0, c.size, items)) if c.size else np.zeros(0, np.int64)
    off = np.zeros(nb + 1, dtype=np.int64)
    carry = 0
    for base in range(0, nb, per_pass):
        part = sums[base:base + per_pass]
        incl = np.cumsum(part)
        off[base:base + part.size] = (0 if drop_carry and base else carry) + incl - part
        carry = (0 if drop_carry and base else carry) + int(incl[-1])
    off[nb] = carry
    out = np.empty(c.size + 1, dtype=np.int64)
    blk = np.repeat(np.arange(nb), items)[:c.size]
    within = np.cumsum(c) - c - np.repeat(np.cumsum(sums) - sums, items)[:c.size]
    out[:-1] = off[blk] + within
    out[-1] = off[nb]
    return out


# ------------------------------------------------------------------------------------------------
# CPU tests
# ------------------------------------------------------------------------------------------------
def _built():
    path = _lib_path()
    if not os.path.exists(path):
        pytest.fail(f"{path} is not built")
    return path


def test_case_table_matches_library():
    built = library_kernels(_built(), FAMILIES)
    table = set(TABLE)
    assert built == table, {"compiled without a case": sorted(built - table),
                            "case without a kernel": sorted(table - built)}
    assert len(table) == 84
    assert len(CASE_IDS) == len(set(CASE_IDS))


def test_three_tables_close_over_the_library():
    """Every dva:: kernel of the library is in exactly one of the three tables."""
    everything = all_library_kernels(_built())
    tables = [set(KM.CASE_IDS), set(PG.CASE_IDS), set(TABLE)]
    union = set().union(*tables)
    assert sum(len(t) for t in tables) == len(union), "a kernel is in two tables"
    assert everything == union, {"in no table": sorted(everything - union), "not in the library": sorted(union - everything)}


def test_every_bucket_index_user_has_a_large_case():
    for user, (small, big) in BK_USERS.items():
        for k in ("bk::scan_block_sums", "bk::scan_of_sums", "bk::scan_apply"):
            assert small in TABLE[k] and big in TABLE[k], (user, k)


def test_parse_nested_functor_names():
    n = "void dva::bk::count_keys<4, dva::det::PixelKey<int, true> >(dva::det::PixelKey<int, true>, long, long, int*)"
    assert canonical(n) == "bk::count_keys<4, dva::det::PixelKey<int, true>"
    assert parse_kernel("dva::bk::scan_of_sums(long*, long)") == ("bk::scan_of_sums", ())


def test_scan_restatement_and_dropped_carry():
    """The restated scan equals the exclusive prefix sum past SCAN_CARRY_BUCKETS buckets; dropping the carry
    between passes of bk::scan_of_sums breaks it."""
    rng = np.random.default_rng(0)
    c = rng.integers(0, 3, SCAN_CARRY_BUCKETS + 400_000)
    want = np.concatenate([[0], np.cumsum(c)])
    assert np.array_equal(scan_exclusive(c), want)
    assert not np.array_equal(scan_exclusive(c, drop_carry=True), want)
    small = c[:100_000]                           # one pass: the bug cannot show below the threshold
    assert np.array_equal(scan_exclusive(small, drop_carry=True), np.concatenate([[0], np.cumsum(small)]))


def test_rank_sort_ties_to_the_later_source_break_the_mapping():
    """Buckets of 32 and 33 equal keys (the register / re-read switch of bk::warp_rank_sort): a rank sort that
    breaks ties by the later source changes the order the stable lexsort reference gives."""
    for L in (32, 33):
        pid = np.zeros(L, dtype=np.int64)
        iid = np.zeros(L, dtype=np.int64)
        src = np.arange(L)
        good = np.lexsort((src, iid, pid))
        bad = np.lexsort((-src, iid, pid))
        assert np.array_equal(good, src) and not np.array_equal(bad, good)


def test_knn_off_by_one_breaks_bit_equality():
    from oracle.neighborhood_oracle import knn_bruteforce
    rng = np.random.default_rng(1)
    p = rng.random((500, 3)).astype(np.float32)
    for k in (1, 64, 65):
        n_ref, d_ref = knn_bruteforce(p, k)
        n_bad, d_bad = knn_bruteforce(p, k + 1)
        n_bad[:, k - 1] = n_bad[:, k]          # the k-th entry taken one position late
        assert not np.array_equal(n_bad[:, :k], n_ref)


def test_zbuffer_tie_to_higher_index_is_caught():
    from oracle import visibility_oracle as VO
    rng = np.random.default_rng(2)
    m, W, H = 4000, 64, 32
    xp, yp = rng.uniform(0, W, m), rng.uniform(0, H, m)
    dist = rng.uniform(1, 5, m).astype(np.float32)
    dist[1::2] = dist[0::2]
    xp[1::2], yp[1::2] = xp[0::2], yp[0::2]
    sp = VO.splat_boxes(xp, yp, dist, W, H, voxel=0.05)
    idx, _, _, _ = VO.zbuffer(sp, dist, xp, yp, W, H, exact=True)
    # the higher index of every tied pair wins instead
    swapped = np.arange(m)
    swapped[0::2], swapped[1::2] = np.arange(1, m, 2), np.arange(0, m, 2)
    idx_b, _, _, _ = VO.zbuffer(sp[swapped], dist[swapped], xp[swapped], yp[swapped], W, H, exact=True)
    assert not np.array_equal(np.sort(swapped[idx_b]), np.sort(idx))


@pytest.mark.parametrize("dt", list(DTYPES))
def test_nll_bounds_reject_lse_of_the_wrong_row(dt):
    gen = torch.Generator().manual_seed(3)
    N, K = 400, 13
    counts = torch.randint(0, 4, (N,), generator=gen)
    csr = torch.cat([torch.zeros(1, dtype=torch.long), counts.cumsum(0)])
    V = int(csr[-1])
    x = (3 * torch.randn(V, K, generator=gen)).to(DTYPES[dt])
    lab = torch.randint(0, K, (N,), generator=gen)
    lab[::5] = -1
    ref = nll_reference(x, lab, csr)
    b_loss, b_grad = nll_bounds(ref, K, dt)
    # the correct gradient rounded to the storage type is inside its bound
    assert violations(ref["grad"].to(DTYPES[dt]), ref["grad"], b_grad)[0] == 0
    # lse taken from the next row
    xd = x.double()
    lse = torch.logsumexp(xd, -1).roll(1)
    tgt, cnt = ref["target"], ref["count"]
    bad = torch.exp(xd - lse.view(-1, 1))
    on = tgt != -1
    bad[on, tgt[on]] -= 1
    bad[~on] = 0
    bad = (bad / cnt).to(DTYPES[dt])
    assert violations(bad, ref["grad"], b_grad)[0] > 0
    loss_bad = float(((lse - xd.gather(1, tgt.clamp(min=0).view(-1, 1)).squeeze(1))[on]).mean())
    assert abs(loss_bad - float(ref["loss"])) > b_loss


def test_nll_reference_with_minus_inf_logits():
    """A row with one finite logit has a finite float64 loss; a row of -inf only is NaN."""
    x = torch.tensor([[-float("inf"), 1.0, -float("inf")], [-float("inf")] * 3])
    ref = nll_reference(x, torch.tensor([1, -1]), None)
    assert float(ref["loss"]) == 0.0 and torch.isfinite(ref["grad"][0]).all()
    ref = nll_reference(x, torch.tensor([1, 0]), None)
    assert torch.isnan(ref["loss"])


def test_resample_channel_mixup_is_caught():
    from oracle import image_resample_oracle as IR
    rng = np.random.default_rng(4)
    img = rng.integers(0, 256, (23, 31, 4), dtype=np.uint8)
    ref = IR.resize(img, (17, 11))
    bad_in = img.copy()
    bad_in[..., 3] = img[..., 2]                 # channel 3 read as channel 2
    assert not np.array_equal(IR.resize(bad_in, (17, 11)), ref)


def test_mapping_feature_bound_rejects_a_dropped_item():
    rng = np.random.default_rng(5)
    ap = np.array([0, 1, 3, 6, 40])
    f = rng.random((40, 16)).astype(np.float32)
    ref = np.add.reduceat(f.astype(np.float64), ap[:-1], axis=0) / np.diff(ap)[:, None]
    b = mapping_feature_bound(f, ap, ref)
    assert (np.abs(ref.astype(np.float32) - ref) <= b).all()
    bad = np.add.reduceat(f[:-1].astype(np.float64), ap[:-1], axis=0) / np.diff(ap)[:, None]
    assert (np.abs(bad - ref) > b).any()
