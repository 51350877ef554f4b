/*
 * dva_b200.h -- C ABI of libdva_b200.so: the H100 (sm_90a) multi-view aggregation hot path.
 *
 * Every entry point replaces one operator (or a fused chain of operators) on the reference's
 * path  ImageMapping gather -> per-point ragged attention over views -> softmax-weighted reduce
 * (DeepViewAgg, torch_points3d/modules/multimodal + torch_points3d/core/multimodal).  The
 * "replaces" line of each declaration cites the reference file:line (relative to the reference
 * repository root) whose behaviour the entry point reproduces.
 *
 * Conventions (all entry points)
 *   - extern "C", plain pointers and sizes; no torch / C++ types.
 *   - all data pointers are DEVICE pointers owned by the caller (workspace included); the
 *     library never allocates or frees device memory and keeps no global mutable state.
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*); no internal
 *     synchronisation, never the legacy default stream unless the caller passes it.
 *   - row-major contiguous tensors. CSR pointers are int64 (the reference dtype,
 *     core/multimodal/csr.py:54). Row indices are int32 or int64 (`idx_is_i64`).
 *   - `dtype` selects the storage type of feature tensors (DVA_F32 / DVA_BF16 / DVA_F16);
 *     scores, softmax statistics and all accumulation are fp32.
 *   - return value: 0 = OK; <0 = DVA_E* argument error (nothing was launched);
 *     >0 = cudaError_t of the failed launch.  dva_last_error() gives a thread-local message.
 */
#ifndef DVA_B200_H_
#define DVA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DVA_ABI_VERSION 1

enum { DVA_OK = 0, DVA_EINVAL = -1, DVA_EALIGN = -2, DVA_EUNSUPPORTED = -3 };
enum { DVA_F32 = 0, DVA_BF16 = 1, DVA_F16 = 2 };
/* reduce codes follow BimodalCSRPool._POOLING_MODES order-independent names (pooling.py:36) */
enum { DVA_SUM = 0, DVA_MEAN = 1, DVA_MAX = 2, DVA_MIN = 3 };

int dva_abi_version(void);
const char* dva_last_error(void);
/* number of kernels this library has launched in this process since load (all threads:
 * autograd runs backward from a worker thread); bench.py reports it as gpu_launches. */
int64_t dva_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * T1 / P1  segment_csr                      replaces torch_scatter.segment_csr as used at
 *   pooling.py:63 (BimodalCSRPool), :289,:295,:519,:525 (pools), :628 (DeepSetFeat.f_pool),
 *   :787,:807 (segment_softmax_csr), :851 (segment_gather_csr); image.py:1767.
 *   out[i,:] = reduce_{p in [ptr[i],ptr[i+1])} src[p,:];  EMPTY segment -> 0 for every reduce
 *   (pooling.py:870).  mean divides by max(count,1).  For max/min `arg` (nullable, int64
 *   [n_seg,K]) receives the FIRST arg-max/min row in segment order, or n_items for empty
 *   segments (torch_scatter convention); backward routes the gradient to that row only.
 * ------------------------------------------------------------------------------------------ */
int dva_segment_csr_fwd(const void* src, const int64_t* ptr, void* out, int64_t* arg,
                        int64_t n_seg, int64_t n_items, int64_t K, int reduce, int dtype,
                        void* stream);
/* grad_src[n_items,K] fully written (zeros where no gradient flows). */
int dva_segment_csr_bwd(const void* grad_out, const int64_t* ptr, const int64_t* arg,
                        void* grad_src, int64_t n_seg, int64_t n_items, int64_t K, int reduce,
                        int dtype, void* stream);

/* P8  gather_csr                            replaces pooling.py:813-841
 *   out[p,:] = src[i,:] for p in [ptr[i],ptr[i+1]).  Its backward is segment_csr(sum). */
int dva_gather_csr(const void* src, const int64_t* ptr, void* out, int64_t n_seg,
                   int64_t n_items, int64_t K, int dtype, void* stream);

/* P7  segment_softmax_csr                   replaces pooling.py:758-810
 *   m = segment max (0 if empty); z = (src-m)/(sqrt(count) if scaling); e = exp(z);
 *   out = e / (segment_sum(e) + eps).   src/out [n_items,K]. */
int dva_segment_softmax_csr_fwd(const void* src, const int64_t* ptr, void* out, int64_t n_seg,
                                int64_t n_items, int64_t K, float eps, int scaling, int dtype,
                                void* stream);
/* grad_src = out * (grad_out - sum_seg(out*grad_out)) / (sqrt(count) if scaling) */
int dva_segment_softmax_csr_bwd(const void* out, const void* grad_out, const int64_t* ptr,
                                void* grad_src, int64_t n_seg, int64_t n_items, int64_t K,
                                int scaling, int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * P3 / P4 core: fused CSR-gather + ragged group softmax + weighted sum + gating.
 *   replaces the chain  modules.py:518 (x_mod[idx_sorting] row gather)  ->
 *   pooling.py:285-300 (GroupBimodalCSRPool)  /  pooling.py:515-530 (QKVBimodalCSRPool):
 *     a    = segment_softmax_csr(compat, ptr, scaling=group_scaling)          [V,G]
 *     y    = segment_csr(x[idx] * expand_group_feat(a, G, C), ptr, 'sum')     [N,C]
 *     t    = tanh(relu(gate_w * segment_csr(compat, ptr, 'max') + gate_b))    [N,G]  (if gating)
 *     out  = y * expand_group_feat(t, G, C)
 *   x      [R,C] feature rows (dtype); idx [V] row of x for view v (nullable: identity, R==V)
 *   compat [V,G] fp32; ptr [N+1] int64; gate_w/gate_b [G] fp32 (both null: no gating)
 *   out    [N,C] (dtype)
 *   saved for backward / save_last taps (all nullable except in training):
 *     att [V,G] fp32 attention a;  seg_max [N,G] fp32;  seg_den [N,G] fp32 (sum e + eps);
 *     seg_arg [N,G] int32 = first arg-max view (absolute view id, -1 if empty)
 *   channel->group map: group_sizes(C,G) of pooling.py:737-755 (first C%G groups one wider).
 *   G must be a power of two <= 32 (all shipped configs use 4); otherwise DVA_EUNSUPPORTED and
 *   the host composes the unfused entry points above.
 * ------------------------------------------------------------------------------------------ */
int dva_view_attention_fwd(const void* x, const void* idx, int idx_is_i64, const float* compat,
                           const int64_t* ptr, const float* gate_w, const float* gate_b,
                           void* out, float* att, float* seg_max, float* seg_den,
                           int32_t* seg_arg, int64_t N, int64_t V, int64_t R, int64_t C,
                           int64_t G, int group_scaling, float eps, int dtype, void* stream);

/* Implementation choice of the fused pair (tuning / test knob, process-wide; results are the same
 * up to fp32 summation order): 0 = auto (default; also DVA_VA_PATH=auto|stream|ring|lane in the
 * environment), 1 = streaming kernels (rows in registers, one point per warp at a time),
 * 2 = ring kernels (rows staged in shared memory by async copies across point boundaries, softmax
 * statistics one lane per point; need G == 4 and rows of whole 16-byte chunks, <= 512 bytes --
 * anything else runs on the streaming kernels whatever the setting), 3 = backward on the
 * lane-per-view kernel (groups of <= 32 views per warp: lane per view for the scores, sub-warp per
 * row for the features; G == 4, rows of 4 / 8 / 16 / 32 chunks), forward as in auto.
 * TEST / TUNING ONLY: production callers leave it at 0; the choice is a pure function of the shape. */
int dva_view_attention_set_path(int path);

/* Backward of the chain above.
 *   grad_out [N,C] (dtype) -> grad_x_rows [V,C] (dtype; row v is d/d(x[idx[v]]); when
 *   scatter_rows!=0 and idx!=null it is written to row idx[v] of a [R,C] buffer instead, which
 *   requires idx to be injective, as view_cat_sorting is, image.py:1549-1574),
 *   grad_compat [V,G] fp32 (softmax path + gating arg-max path),
 *   grad_gate [2,G] fp32 (d gate_w ; d gate_b), nullable when no gating.
 *   workspace: dva_view_attention_bwd_workspace_bytes(G) bytes (per-block partials). */
size_t dva_view_attention_bwd_workspace_bytes(int64_t G);
int dva_view_attention_bwd(const void* x, const void* idx, int idx_is_i64, const float* compat,
                           const int64_t* ptr, const float* gate_w, const float* gate_b,
                           const void* grad_out, const float* seg_max, const float* seg_den,
                           const int32_t* seg_arg, void* grad_x_rows, float* grad_compat,
                           float* grad_gate, int scatter_rows, int64_t N, int64_t V, int64_t R,
                           int64_t C, int64_t G, int group_scaling, int dtype, void* workspace,
                           size_t workspace_bytes, void* stream);

/* P4  ragged per-group Q.K scores           replaces pooling.py:499-512
 *   compat[v,g] = scale * sum_d keys[v,g*D+d] * queries[i(v),g*D+d]   (i(v): point of view v;
 *   the reference materialises repeat_interleave(queries), pooling.py:500).  fp32 I/O. */
int dva_qk_scores_fwd(const float* keys, const float* queries, const int64_t* ptr, float* compat,
                      int64_t N, int64_t V, int64_t G, int64_t D, float scale, void* stream);
int dva_qk_scores_bwd(const float* keys, const float* queries, const int64_t* ptr,
                      const float* grad_compat, float* grad_keys, float* grad_queries, int64_t N,
                      int64_t V, int64_t G, int64_t D, float scale, void* stream);

/* P2  HeuristicBimodalCSRPool               replaces pooling.py:129-152
 *   j_i = first arg-max/min over the segment of x_map[:,feat]; out[i,:] = x_mod[j_i,:] or 0.
 *   arg [N] int64 (n_items when empty). */
int dva_heuristic_pool_fwd(const void* x_mod, const float* x_map, int64_t map_stride,
                           int64_t feat, const int64_t* ptr, void* out, int64_t* arg, int64_t N,
                           int64_t V, int64_t C, int use_max, int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * I5 + P1  fused feature-map gather + atomic pool
 *   replaces image.py:1285 (x[(img, ..., py, px)] NCHW advanced-index gather) followed by
 *   modules.py:497-500 -> pooling.py:63 (BimodalCSRPool over the atomic CSR).
 *   fmap [B,C,H,W] (channels_last=0) or [B,H,W,C] (channels_last=1), dtype
 *   img [Vw] int64 image of each view; pix [P,2] (x,y) int16/int32 (pix_is_i16)
 *   aptr [Vw+1] int64 atomic CSR;  out [Vw,C];  arg [Vw,C] int64 pixel slot (nullable, max/min)
 * ------------------------------------------------------------------------------------------ */
int dva_gather_pool_fwd(const void* fmap, int channels_last, const int64_t* img, const void* pix,
                        int pix_is_i16, const int64_t* aptr, void* out, int64_t* arg,
                        int64_t B, int64_t C, int64_t H, int64_t W, int64_t Vw, int64_t P,
                        int reduce, int dtype, void* stream);
/* grad_fmap must be zero-initialised by the caller; gradients are accumulated with fp32
 * atomics when dtype==DVA_F32 (pixel reuse across views), see DESIGN.md. */
int dva_gather_pool_bwd(const void* grad_out, int channels_last, const int64_t* img,
                        const void* pix, int pix_is_i16, const int64_t* aptr, const int64_t* arg,
                        float* grad_fmap, int64_t B, int64_t C, int64_t H, int64_t W, int64_t Vw,
                        int64_t P, int reduce, int dtype, void* stream);

/* Deterministic variant of dva_gather_pool_bwd          replaces the backward of image.py:1285
 *   (x[feature_map_indexing]) + pooling.py:63 under torch.use_deterministic_algorithms(True).
 *   grad_fmap is fully written (zeros included; no zero-initialisation needed).  Every element is the
 *   fp32 sum, from +0.0f, with one round-to-nearest addition per contribution, of the contributions of
 *   its map pixel in ascending pixel-slot order p: g = grad_out[w, c] of the slot's view w;
 *   mean: g / n_w (rounded); max / min: only the slot with arg[w, c] == p (any slot when n_w == 1).
 *   Out-of-range pixels and images are clamped as in the forward.  The result does not depend on
 *   the launch configuration.  Needs fewer than 2^31 views.
 *   workspace: dva_gather_pool_bwd_det_workspace_bytes(B, H, W, P) bytes (pixel-bucket index). */
size_t dva_gather_pool_bwd_det_workspace_bytes(int64_t B, int64_t H, int64_t W, int64_t P);
int dva_gather_pool_bwd_det(const void* grad_out, int channels_last, const int64_t* img,
                            const void* pix, int pix_is_i16, const int64_t* aptr, const int64_t* arg,
                            float* grad_fmap, int64_t B, int64_t C, int64_t H, int64_t W, int64_t Vw,
                            int64_t P, int reduce, int dtype, void* workspace, size_t workspace_bytes,
                            void* stream);

/* [B,R,S] -> [B,S,R] layout change (dtype-sized elements), e.g. the reference's NCHW-contiguous
 * feature maps (image.py:1884 indexes them as x[b, :, y, x]) to channels-last and map gradients back,
 * so that dva_gather_pool_* / dva_interp_pool_* can run their 16-byte-chunk channels-last kernels. */
int dva_transpose_last2(const void* src, void* dst, int64_t B, int64_t R, int64_t S, int dtype, void* stream);

/* I5b  bilinear variant: the `interpolate=True` branch of get_mapped_features
 *   replaces image.py:1278-1283 -> sparse_interpolation (image.py:105-170, padding 'border')
 *   followed by the same atomic pool.  pix are at the MAPPING resolution (map_w, map_h); every
 *   pixel reads the 4 bilinear corners of the replicate-padded [H,W] map.  The fp32 operation
 *   order is the reference's, so fp32 results (and max / argmax choices) are identical.
 *   A per-pixel interpolation without pooling is aptr = 0..P with reduce = DVA_SUM. */
int dva_interp_pool_fwd(const void* fmap, int channels_last, const int64_t* img, const void* pix,
                        int pix_is_i16, const int64_t* aptr, void* out, int64_t* arg,
                        int64_t B, int64_t C, int64_t H, int64_t W, int64_t map_w, int64_t map_h,
                        int64_t Vw, int64_t P, int reduce, int dtype, void* stream);
int dva_interp_pool_bwd(const void* grad_out, int channels_last, const int64_t* img,
                        const void* pix, int pix_is_i16, const int64_t* aptr, const int64_t* arg,
                        float* grad_fmap, int64_t B, int64_t C, int64_t H, int64_t W,
                        int64_t map_w, int64_t map_h, int64_t Vw, int64_t P, int reduce, int dtype,
                        void* stream);

/* Deterministic variant of dva_interp_pool_bwd          replaces the backward of image.py:1278-1283
 *   (sparse_interpolation, image.py:105-170) + pooling.py:63 under torch.use_deterministic_algorithms(True).
 *   As dva_gather_pool_bwd_det with four contributions per slot, in the order (p, k), k = corners
 *   top-left, top-right, bottom-left, bottom-right; a contribution is the rounded product of the
 *   corner weight and the value above (two corners clamped onto one pixel stay two contributions).
 *   workspace: dva_interp_pool_bwd_det_workspace_bytes(B, H, W, P) bytes. */
size_t dva_interp_pool_bwd_det_workspace_bytes(int64_t B, int64_t H, int64_t W, int64_t P);
int dva_interp_pool_bwd_det(const void* grad_out, int channels_last, const int64_t* img,
                            const void* pix, int pix_is_i16, const int64_t* aptr, const int64_t* arg,
                            float* grad_fmap, int64_t B, int64_t C, int64_t H, int64_t W,
                            int64_t map_w, int64_t map_h, int64_t Vw, int64_t P, int reduce, int dtype,
                            void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * N1  neighbourhood-based mapping features (density, occlusion)
 *   replaces NeighborhoodBasedMappingFeatures._process,
 *   core/data_transform/multimodal/image.py:483-612 (KeOps argKmin branch :504-514; the FAISS
 *   branch is approximate and not reproduced).
 *   dva_knn_cell_ids : cell[i] = linear cell of point i in a gx x gy x gz grid of `cell_size`
 *                      cubes anchored at (ox,oy,oz) (clamped).  The caller sorts points by cell
 *                      and builds cell_ptr [gx*gy*gz+1] (dva_csr_pointers_from_sorted).
 *   dva_knn_grid     : exact k nearest neighbours (self included), 1 <= k <= 128 (else
 *                      DVA_EUNSUPPORTED, nothing launched), of every point among all points;
 *                      squared distance (dx*dx + dy*dy) + dz*dz in fp32, ties by index.  Planar
 *                      inputs (z = 0) give the exact 2D squared distance (image-plane k-NN).
 *                      neighbors [n,k] int64 and dist2 [n,k] (nullable) are indexed by
 *                      ORIGINAL point id, ascending (dist2, id).
 *   dva_knn_query    : the same search for a query set among a separate search set; replaces the
 *                      KeOps brute-force `argmin` of models/segmentation/multimodal/no3d.py:105-125
 *                      (nearest seen point of every unseen point).  The grid (origin, cell_size,
 *                      gx x gy x gz) is built over the search set: search_sorted / search_order /
 *                      cell_ptr as for dva_knn_grid.  Queries are cell-sorted too: query_cell_sorted
 *                      from dva_knn_cell_ids on the same grid (clamped, so queries outside it fall in
 *                      a border cell), query_order [nq] their original ids.  block_counts
 *                      [ceil(gz/8)*ceil(gy/8)*ceil(gx/8)] int32 = search points per block of 8^3
 *                      cells: a query still open after 6 fine shells walks shells of non-empty
 *                      blocks, so far queries do not scan the search set.  Same arithmetic and tie
 *                      order as dva_knn_grid; neighbors [nq,k] (search ids) and dist2 (nullable) are
 *                      indexed by ORIGINAL query id.  nq == 0 launches nothing; ns < k is DVA_EINVAL.
 *   dva_neighborhood_features : out [V, nk*(density + occlusion)] fp32 = for every k of the
 *                      ascending klist: density of the view's point ((k+1)/(3.1416 d_k^2)/(1/voxel^2),
 *                      NaN -> 1, :527-537), then occlusion of the view ((1 + #neighbours seen by
 *                      the view's image)/(k+1), :563-584).  view_ptr [N+1] / images [V]: the view
 *                      CSR; view_point [V] = point of each view.
 * ------------------------------------------------------------------------------------------ */
int dva_knn_cell_ids(const float* xyz, int64_t* cell, int64_t n, float ox, float oy, float oz,
                     float cell_size, int gx, int gy, int gz, void* stream);
int dva_knn_grid(const float* xyz_sorted, const int64_t* cell_sorted, const int64_t* order,
                 const int64_t* cell_ptr, int64_t n, int k, float ox, float oy, float oz,
                 float cell_size, int gx, int gy, int gz, int64_t* neighbors, float* dist2,
                 void* stream);
int dva_knn_query(const float* query_sorted, const int64_t* query_cell_sorted, const int64_t* query_order,
                  int64_t nq, const float* search_sorted, const int64_t* search_order,
                  const int64_t* cell_ptr, const int32_t* block_counts, int64_t ns, int k, float ox,
                  float oy, float oz, float cell_size, int gx, int gy, int gz, int64_t* neighbors,
                  float* dist2, void* stream);
int dva_neighborhood_features(const float* xyz, const int64_t* neighbors, int kmax,
                              const int64_t* view_ptr, const int64_t* images,
                              const int64_t* view_point, const int32_t* klist, int nk,
                              double voxel, int density, int occlusion, float* out, int64_t N,
                              int64_t V, void* stream);

/* ------------------------------------------------------------------------------------------
 * P9  dense projection GEMM of an MLP layer (wgmma / TMA / mbarrier)
 *   replaces the nn.Linear(bias=False) of base_modules.py:42 in every pool MLP.
 *   layout 0: D[M,N] = A[M,K] . B[N,K]^T   (forward,  B = weight [out,in])
 *   layout 1: D[M,N] = A[M,K] . B[K,N]     (backward, dX = dZ . weight)
 *   layout 2: D[N,K] = A[M,N]^T . B[M,K]   (backward, dW = dZ^T . X; stream-K over the M rows)
 *   fp32 row-major operands.  Two kernel families behind the one entry point:
 *     N <= 64 and K <= 64 (any values; every MLP of the map encoders, pooling.py:645-656): "skinny"
 *       kernels -- weights in shared memory, 128-row tiles double-buffered by cp.async, coalesced
 *       16-byte global traffic, 3xTF32 split operands on mma.sync (fp32-grade accuracy, ~1e-6), dW
 *       as per-CTA partials reduced in a fixed order (deterministic);
 *     otherwise the hand-written wgmma kernels of csrc/tc_gemm.cu (TMA-fed wgmma.mma_async tf32,
 *       register accumulators, 3xTF32 split operands: ~1e-6 of the result's max against fp64; dW as
 *       per-CTA partial tiles reduced in a fixed order): operands 16-byte aligned, N % 4 == 0 and
 *       K % 4 == 0 (else DVA_EUNSUPPORTED; ops.linear zero-pads such widths).
 *   `precision` is accepted for ABI stability (0 or 1) and ignored: every path is fp32-grade.
 *   workspace: dva_linear_gemm_workspace_bytes().  dva_linear_gemm_skinny(): 1 when the skinny kernels
 *   serve the shape (any operand alignment), 0 when the wgmma kernels do (16-byte aligned operands).
 * ------------------------------------------------------------------------------------------ */
int dva_linear_gemm_skinny(int64_t M, int64_t N, int64_t K, int layout);
size_t dva_linear_gemm_workspace_bytes(int64_t M, int64_t N, int64_t K, int layout, int precision);
int dva_linear_gemm(const float* A, const float* B, float* D, int64_t M, int64_t N, int64_t K, int layout,
                    int precision, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * P9  Linear with the BatchNorm batch statistics taken in the GEMM epilogue
 *   replaces base_modules.py:42-44 (nn.Linear(bias=False) followed by the statistics half of
 *   FastBatchNorm1d) for the wide layers (E_mod, E_mix, E_main): D[M,n_out] = X[M,k_red] . W[n_out,k_red]^T
 *   by the wgmma rows kernel, whose epilogue accumulates each column's shifted sum / sum of squares
 *   from the accumulator registers while storing (fp64 per CTA in shared memory); a one-warp-per-column kernel combines the per-CTA
 *   partials in fp64 (fixed order) into mean / invstd [n_out] (biased variance) and updates the running
 *   buffers (momentum, unbiased variance) like nn.BatchNorm1d.  The apply half is dva_bn_act_fwd with
 *   training = 0 on these mean / invstd.  supported(): 32 <= n_out <= 128, n_out % 4 == 0, k_red >= 8,
 *   k_red % 4 == 0 (the shapes dva_linear_gemm serves with the wgmma rows kernel; with DVA_TC_NARROW=0 in the
 *   environment only n_out > 32 and k_red > 32, the round-1 routing); else DVA_EUNSUPPORTED.
 * ------------------------------------------------------------------------------------------ */
int dva_linear_bnstats_supported(int64_t M, int64_t n_out, int64_t k_red);
size_t dva_linear_bnstats_workspace_bytes(int64_t n_out, int64_t k_red);
int dva_linear_bnstats_fwd(const float* X, const float* W, float* D, int64_t M, int64_t n_out, int64_t k_red,
                           float eps, float momentum, float* mean, float* invstd, float* running_mean,
                           float* running_var, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * P9  fused BatchNorm1d (+ LeakyReLU) of an MLP layer
 *   replaces core/common_modules/base_modules.py:38-48 (Linear -> FastBatchNorm1d -> LeakyReLU(0.2))
 *   after the Linear, and FastBatchNorm1d._forward_sparse :139-148: per-column batch statistics
 *   over ALL rows in training (biased variance for normalisation, unbiased for running_var,
 *   momentum update), y = act(gamma * (z - mean) * invstd + beta), act(a) = a > 0 ? a : slope * a
 *   (slope = 1: plain BatchNorm).  z, y [R,C] (dtype); gamma/beta nullable; mean/invstd [C] fp32 are
 *   written in training and READ in eval (host passes running_mean and rsqrt(running_var + eps)).
 *   Backward: dz [R,C] (NULL: statistics pass only); dbeta_dgamma [2,C] fp32 = (sum g ; sum g * zhat) with g = dy * act'.
 *   workspace: dva_bn_workspace_bytes(R, C) bytes (per-CTA partial sums, deterministic).
 * ------------------------------------------------------------------------------------------ */
size_t dva_bn_workspace_bytes(int64_t R, int64_t C);
int dva_bn_act_fwd(const void* z, const float* gamma, const float* beta, float* running_mean,
                   float* running_var, float* mean, float* invstd, void* y, int64_t R, int64_t C,
                   float eps, float momentum, float slope, int training, int dtype, void* workspace,
                   size_t workspace_bytes, void* stream);
int dva_bn_act_bwd(const void* dy, const void* z, const float* gamma, const float* beta,
                   const float* mean, const float* invstd, void* dz, float* dbeta_dgamma, int64_t R,
                   int64_t C, float slope, int training, int dtype, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * P9 / P5  backward of one narrow MLP layer  a = LeakyReLU(BatchNorm1d(x . W^T))   (training statistics)
 *   replaces the autograd chain of base_modules.py:38-48 for the layers of the map encoders
 *   (DeepSetFeat / MLPSetFeat, pooling.py:645-656, 686: 8 / 32 / 64 -> 32 on one row per view):
 *   pass 1 = the statistics half of dva_bn_act_bwd (dz = NULL there: reduction only), pass 2 = ONE kernel that
 *   forms dz = gamma invstd (g - mean(g) - zhat mean(g zhat)) on chip and emits dX = dz . W and dW = dz^T . x
 *   from the same tile (3xTF32 mma.sync, fp32-grade): 3 reads + 1 write of the rows instead of 5 + 2.
 *   dA, Z [M,N] fp32 (gradient of the layer output, saved pre-BatchNorm linear output); X [M,K] fp32 layer input;
 *   W [N,K]; gamma / beta nullable; mean / invstd [N] of the forward; dX [M,K] nullable (first layer);
 *   dW [N,K]; dbeta_dgamma [2,N] = (sum g ; sum g zhat).  supported(): N <= 32, K <= 64, both % 4 == 0.
 *   Row pointers 16-byte aligned.  Deterministic (per-CTA partials summed in a fixed order).
 * ------------------------------------------------------------------------------------------ */
int dva_mlp_layer_bwd_supported(int64_t M, int64_t N, int64_t K);
size_t dva_mlp_layer_bwd_workspace_bytes(int64_t M, int64_t N, int64_t K);
int dva_mlp_layer_bwd(const float* dA, const float* Z, const float* X, const float* W, const float* gamma,
                      const float* beta, const float* mean, const float* invstd, float* dX, float* dW,
                      float* dbeta_dgamma, int64_t M, int64_t N, int64_t K, float slope, void* workspace,
                      size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Z3  z-buffer visibility from splatting    replaces visibility.py:1073-1195 (CPU/numba oracle)
 *   splat [m,4] int32 (x_a,x_b,y_a,y_b) already clamped, y relative to the un-cropped image;
 *   dist [m] fp32.  Point i wins pixel (x,y) iff dist is the smallest, ties -> lowest i
 *   (strict '<' while iterating ascending, visibility.py:1148-1162) -- realised as one
 *   64-bit atomicMin on (dist_bits<<32 | i).
 *   zbuf [W*Hc] uint64 workspace (Hc = H - crop_top - crop_bottom), initialised by the call.
 *   exact==0: idx_map [W*Hc] int64 (-1 = empty) holds the winning point per pixel.
 *   exact!=0: idx_map re-rasterised with splat centres only: (int(x_proj), int(y_proj)-crop_top),
 *             highest seen index wins a shared centre (visibility.py:1168-1187).
 *   x_proj/y_proj [m] fp64 (numba returns float64, visibility.py:252).
 * ------------------------------------------------------------------------------------------ */
int dva_zbuffer_splat(const int32_t* splat, const float* dist, const double* x_proj,
                      const double* y_proj, unsigned long long* zbuf, int64_t* idx_map,
                      uint8_t* seen, int64_t m, int64_t W, int64_t H, int64_t crop_top,
                      int64_t crop_bottom, int exact, void* stream);

/* Z2  splat boxes                           replaces visibility.py:630-704 (equirectangular),
 *   :761-827 (pinhole).  camera: 0 = s3dis_equirectangular, 1 = pinhole (fx, fy given).
 *   numba evaluates these expressions in float64 (float32 array x Python float), hence the
 *   double parameters.  Output splat [m,4] int32 (16-byte aligned), clamped to the (cropped)
 *   image like the reference; y is relative to the un-cropped image. */
int dva_splat_boxes(const double* x_proj, const double* y_proj, const float* dist,
                    int32_t* splat, int64_t m, int64_t W, int64_t H, int64_t crop_top,
                    int64_t crop_bottom, double voxel, double k_swell, double d_swell, int camera,
                    double fx, double fy, void* stream);

/* Z2  splat boxes from explicit widths        replaces the rounding / clamping tail of
 *   fisheye_splat_cpu (visibility.py:916-951); width [m] fp64 = 2*|proj(xyz) - proj(xyz + dz)|
 *   (visibility.py:903-914) is produced by the host mirror with two dva_project_camera calls. */
int dva_splat_boxes_from_width(const double* x_proj, const double* y_proj, const double* width,
                               int32_t* splat, int64_t m, int64_t W, int64_t H, int64_t crop_top,
                               int64_t crop_bottom, void* stream);

/* Z1  equirectangular camera projection      replaces visibility.py:150-182 + :509-513 + :395-435
 *   xyz [n,3] fp32; img_pose [12] fp32 on device = camera position (3) followed by the 3x3
 *   rotation matrix of pose_to_rotation_matrix (visibility.py:57-90), row-major, computed by the
 *   host mirror.  Outputs dist [n] fp32, x_proj,y_proj [n] fp64, keep [n] uint8 = in
 *   (r_min,r_max) and inside the (cropped) field of view (no image mask). */
int dva_project_equirectangular(const float* xyz, const float* img_pose, float* dist,
                                double* x_proj, double* y_proj, uint8_t* keep, int64_t n,
                                int64_t W, int64_t H, int64_t crop_top, int64_t crop_bottom,
                                float r_min, float r_max, void* stream);

/* Z1  pinhole / fisheye camera projection    replaces visibility.py:219-252 (pinhole_projection_cpu,
 *   cameras 'scannet' and 'kitti360_perspective'), :288-339 (fisheye_projection_cpu,
 *   'kitti360_fisheye') + the range / field-of-view filter of camera_projection_cpu :509-536.
 *   cam [26] fp32 on device = img_xyz(3), A(9 row-major), t0(3), t1(3), intr(8) with
 *   p = A (xyz - t0) + t1  (scannet: A,t1 from inv(extrinsic), t0 = 0; kitti360: A = R^T, t0 = T);
 *   camera 1 = pinhole (intr = fx, fy, cx, cy), 3 = fisheye (intr = xi,k1,k2,gamma1,gamma2,u0,v0). */
int dva_project_camera(const float* xyz, const float* cam, int camera, float* dist, double* x_proj,
                       double* y_proj, uint8_t* keep, int64_t n, int64_t W, int64_t H,
                       int64_t crop_top, int64_t crop_bottom, float r_min, float r_max, void* stream);

/* rows scatter-add: dst[idx[v], :] += src[v, :] for v < V; dst [R, C] fp32 must be zero-initialised by the
 * caller; rows with idx outside [0, R) are skipped.  Backward of `x_mod[row_index]` when row_index repeats
 * rows (modules.py:518 with a caller-supplied index) and of HeuristicBimodalCSRPool's row pick
 * (pooling.py:146-150, "no view" = index V). */
int dva_scatter_add_rows(const void* src, const int64_t* idx, float* dst, int64_t V, int64_t R, int64_t C,
                         int dtype, void* stream);
/* Deterministic variant of dva_scatter_add_rows          replaces the same two backwards (modules.py:518,
 *   pooling.py:146-150) under torch.use_deterministic_algorithms(True): dst [R, C] fp32 is fully written;
 *   row r is the fp32 sum, from +0.0f in ascending v, of src[v] over the v with idx[v] == r.
 *   workspace: dva_scatter_add_rows_det_workspace_bytes(V, R) bytes (row-bucket index). */
size_t dva_scatter_add_rows_det_workspace_bytes(int64_t V, int64_t R);
int dva_scatter_add_rows_det(const void* src, const int64_t* idx, float* dst, int64_t V, int64_t R, int64_t C,
                             int dtype, void* workspace, size_t workspace_bytes, void* stream);

/* I1 / I4 / I6  native construction of the point -> view -> pixel CSR (csrc/mapping_build.cu)
 *   replaces ImageMapping.from_dense image.py:1728-1795 (lexargsort + unique + cumsum chains) and the
 *   dense expansion / lexargunique / scatter_mean / from_dense sequence of select_points('merge')
 *   image.py:2211-2273.  Items i = 0..n-1: (point_ids[i] in [0, num_points), image_ids[i], pixels[i] = (x, y)
 *   as int16 / int32 / int64 pairs: pix_code 0 / 1 / 2).  Items are bucketed by point (histogram, scan,
 *   scatter) and every point's items ordered by (image, source index) -- or, with dedupe_pixels,
 *   by (image, x, y, source index; 0 <= x, y < 65536) dropping repeated (image, x, y).  Outputs, all
 *   preallocated by the caller with n (resp. n + 1) rows: view_ptr [num_points + 1], images_out [V],
 *   atomic_ptr [V + 1], pixels_out [P, 2] (same integer type), feat_out [V, F] = mean of
 *   feat[feat_row ? feat_row[i] : i] over the view's items with feat_on[i] != 0 (nullable: all), F <= 16;
 *   order_out [P] (nullable) = source item of every kept pixel; counts [3] (device) = V, P, status
 *   (status bit 0: a point id was out of range; such items are skipped).  Deterministic = the result of a
 *   stable lexicographic sort.  Nothing is read back: the caller reads `counts` once to slice the outputs.
 *   dva_view_cat_sorting: ImageData.view_cat_sorting / view_cat_csr_indexing image.py:1549-1588 for S
 *   settings over the same N points in closed form (no argsort): ptrs = device array of S device pointers
 *   to the settings' view pointers [N + 1], bases[s] = views of the settings before s. */
size_t dva_mapping_build_workspace_bytes(int64_t n_items, int64_t num_points);
int dva_mapping_build(const int64_t* point_ids, const int64_t* image_ids, const void* pixels, int pix_code,
                      const float* feat, const int64_t* feat_row, const uint8_t* feat_on, int64_t F,
                      int64_t n_items, int64_t num_points, int dedupe_pixels, int64_t* view_ptr,
                      int64_t* images_out, int64_t* atomic_ptr, void* pixels_out, float* feat_out,
                      int64_t* order_out, int64_t* counts, void* workspace, size_t workspace_bytes, void* stream);
int dva_view_cat_sorting(const int64_t* const* ptrs, const int64_t* bases, int64_t S, int64_t N,
                         int64_t* sorting, int64_t* csr_cat, void* stream);

/* T1  per-image mapping statistics (csrc/image_transforms.cu)     replaces the torch_scatter passes of
 *   PickImagesFromMappingArea, ImageMapping.bounding_boxes (CropImageGroups) and CenterRoll
 *   (core/data_transform/multimodal/image.py:733-749, :999-1015).  Views v < V: images [V] int64 in
 *   [0, n_img) (others skipped), atomic_ptr [V + 1], pixels [P, 2] (x, y) int16 / int32 / int64 (pix_code
 *   0 / 1 / 2).  Outputs: count [n_img] int64 pixels per image; bbox [n_img, 4] int32 = (x_min, x_max,
 *   y_min, y_max), all 0 for an image without pixels; occ [n_img, 8] uint32 (nullable) = bit q set for
 *   every q = (int64)(fp32(fp32(x * 256) / ref_w)) & 255 of the image.  Integer atomics only: the result
 *   does not depend on the launch. */
int dva_mapping_image_stats(const int64_t* images, const int64_t* atomic_ptr, const void* pixels, int pix_code,
                            int64_t V, int64_t n_img, int64_t ref_w, int64_t* count, int32_t* bbox, uint32_t* occ,
                            void* stream);

/* T2  CenterRoll cost                          replaces image.py:1009-1029 on the occupancy of T1.
 *   Candidate rolls r = 0, s, 2s, .. < 256 with s = 256 / angular_res (integer division); bins (b + r) & 255;
 *   cost = (w_max - w_min) + int(|fp32(w_max + w_min) / 2 - 128|), first least cost wins;
 *   rollings [n_img] int64 = (int64)(fp32(r / 256) * ref_w). */
int dva_center_roll(const uint32_t* occ, int64_t n_img, int angular_res, int64_t ref_w, int64_t* rollings,
                    void* stream);

/* T3  batched feature-map remap                 replaces the per-image roll / slice / flip loops + torch.cat
 *   of SameSettingImageData.update_rollings / update_cropping and RandomHorizontalFlip (image.py:605-609,
 *   :709-714, data_transform image.py:1207-1212).  in [B, C, Hi, Wi], out [B, C, Ho, Wo], both NCHW or both
 *   channels-last (channels_last != 0), elements of elem_bytes = 1, 2 or 4 bytes moved as raw bytes:
 *     out[b, c, y, x] = in[b, c, oy_b + y, (ox_b + (flip ? Wo - 1 - x : x) - r_b) mod Wi]
 *   rolls [B] int64 (nullable: 0), offsets [B, 2] int64 (ox, oy) (nullable: 0).  Rows whose oy_b + y falls
 *   outside the input are written as zeros. */
int dva_image_remap(const void* in, void* out, int64_t B, int64_t C, int64_t Hi, int64_t Wi, int64_t Ho, int64_t Wo,
                    int elem_bytes, int channels_last, const int64_t* rolls, const int64_t* offsets, int flip,
                    void* stream);

/* T4  coverage bookkeeping of PickImagesFromMemoryCredit      replaces the dense bool[n_img, N] table and
 *   the per-pick logical_and loop of image.py:804-867.  Views v < V of all settings: gimg [V] = global image id
 *   in [0, n_img) (setting base + local id), vpoint [V] = point id in [0, N).  dva_coverage_index builds the
 *   image -> points and point -> images lists in the workspace (dva_coverage_index_workspace_bytes) and sets
 *   unseen [n_img] int32 = views of every image, seen [N] int32 = 0.  dva_coverage_pick(g): every point p of
 *   image g with atomicExch(&seen[p], 1) == 0 takes one off unseen[j] of every image j that sees p.  Integer
 *   counts: the result does not depend on the order.  Total work over all picks <= V. */
size_t dva_coverage_index_workspace_bytes(int64_t V, int64_t n_img, int64_t N);
int dva_coverage_index(const int64_t* gimg, const int64_t* vpoint, int64_t V, int64_t n_img, int64_t N,
                       int32_t* unseen, int32_t* seen, void* workspace, size_t workspace_bytes, void* stream);
int dva_coverage_pick(int64_t g, int64_t V, int64_t n_img, int64_t N, int32_t* unseen, int32_t* seen,
                      const void* workspace, size_t workspace_bytes, void* stream);

/* I1  Pillow-exact image resize                 replaces PIL.Image.resize(size, box=...) (BICUBIC, 8 bits) of
 *   SameSettingImageData.read_images (image.py:1061, :1093).  in [B, Hi, Wi, C] uint8 (channels-last, 1 <= C <= 4),
 *   out [B, Ho, Wo, C] uint8.  Tables from the caller: bounds [n_out, 2] int32 = (first source index, count) and
 *   coef [n_out, k] int32 weights scaled by 2^22 (Pillow's precompute_coeffs + normalize_coeffs_8bpc), shared by
 *   all images or per image (x_per_image / y_per_image: [B, n_out, ...]).  Horizontal pass (xcoef non-null):
 *   tmp[b, t, x] over source rows yfirst[b] + t, t < T (rows >= Hi skipped; yfirst nullable: 0); the vertical
 *   bounds are then relative to yfirst[b].  Vertical pass (ycoef non-null) reads tmp [B, T, Wo, C], or `in`
 *   when there is no horizontal pass (Wo == Wi); with no vertical pass the horizontal one writes `out` (T == Ho).
 *   Every sum starts at 2^21, accumulates in int32, is shifted right by 22 and clamped to [0, 255] (uint8
 *   between the passes, as Pillow clips).  Integer only: the result does not depend on the launch. */
int dva_resample_u8(const uint8_t* in, uint8_t* tmp, uint8_t* out, int64_t B, int64_t Hi, int64_t Wi, int64_t C,
                    int64_t Ho, int64_t Wo, int64_t T, const int32_t* xbounds, const int32_t* xcoef, int64_t kx,
                    int x_per_image, const int32_t* ybounds, const int32_t* ycoef, int64_t ky, int y_per_image,
                    const int32_t* yfirst, void* stream);

/* I2  non-static pixel mask                     replaces the per-image comparison loop of NonStaticMask
 *   (data_transform image.py:139-154).  imgs [n, H, W, C] uint8 channels-last, n >= 2; mask [W, H] bytes 0 / 1 (a torch.bool buffer):
 *     mask[x, y] = OR over i >= 1 of AND over c of (imgs[i, y, x, c] != imgs[0, y, x, c]) */
int dva_nonstatic_mask(const uint8_t* imgs, int64_t n, int64_t H, int64_t W, int64_t C, uint8_t* mask, void* stream);

/* I3  colour jitter on uint8 images             replaces torchvision's ColorJitter.forward as the reference's
 *   ColorJitter calls it (data_transform image.py:1249-1259), i.e. _functional_tensor.adjust_brightness /
 *   adjust_contrast / adjust_saturation over _blend and rgb_to_grayscale, for drawn factors (no hue).
 *   in, out [B, 3, H, W] uint8, both NCHW or both channels-last (channels_last != 0), any H and W.  Ops i < n_ops
 *   (0 <= n_ops <= 3) in that order, op code i in bits 4i..4i+3 of op_codes (0 brightness, 1 contrast,
 *   2 saturation, each at most once), factor ratio_i >= 0 and rest_i = fp32(1 - ratio_i) (float64 subtraction).
 *   Per op and channel, in fp32 without contraction:
 *     v' = trunc(clamp(ratio * v + rest * o, 0, 255)),  o = 0 (brightness), the pixel's grayscale (saturation),
 *     or the image's contrast mean;  grayscale = trunc((0.2989 r + 0.587 g) + 0.114 b).
 *   Contrast mean = fp32(double(S) / double(H W)), S the exact sum of the grayscale bytes of the image after the
 *   ops before contrast (torchvision's fp32 torch.mean may differ by an ulp).  With contrast, a first pass sums S
 *   into the workspace (dva_color_jitter_u8_workspace_bytes(B) bytes, zeroed on the stream by the call); the apply
 *   pass reads it on the device.  Integer sums: the result does not depend on the launch. */
size_t dva_color_jitter_u8_workspace_bytes(int64_t B);
int dva_color_jitter_u8(const uint8_t* in, uint8_t* out, int64_t B, int64_t H, int64_t W, int channels_last,
                        int n_ops, int op_codes, float ratio0, float rest0, float ratio1, float rest1, float ratio2,
                        float rest2, void* workspace, size_t workspace_bytes, void* stream);

/* I4  ToFloatImage / Normalize                   replaces `images.x.float() / 255` (data_transform
 *   image.py:1221-1232) and torchvision's _functional_tensor.normalize, `sub_(mean).div_(std)` with fp32
 *   [C, 1, 1] tensors, as the reference's Normalize calls it (:1271-1282).  in [B, C, H, W] uint8 (in_u8 != 0)
 *   or fp32, out [B, C, H, W] fp32, both NCHW or both channels-last, 1 <= C <= 4:
 *     out = (fp32(in) - m_c) / s_c   with true division (ToFloatImage: m_c = 0, s_c = 255).
 *   The channel statistics are passed by value (unused ones ignored): no copy to the device. */
int dva_image_to_float(const void* in, int in_u8, float* out, int64_t B, int64_t C, int64_t H, int64_t W,
                       int channels_last, float m0, float m1, float m2, float m3, float s0, float s1, float s2,
                       float s3, void* stream);

/* L1  log-softmax NLL over a view CSR           replaces models/segmentation/multimodal/no3d.py:144-154
 *   F.nll_loss(F.log_softmax(head(last_view_x_mod)), repeat_interleave(labels, counts), ignore_index=-1),
 *   mean reduction, without the [V] target and [V, K] log-prob tensors.  logits [V, K] (fp32 / bf16 / fp16
 *   storage, fp32 math, 1 <= K <= 64, else DVA_EUNSUPPORTED), labels [N] int64, csr_idx [N+1] int64 (view v
 *   belongs to point p for csr_idx[p] <= v < csr_idx[p+1]) or NULL for V == N (one view per point).
 *   A view counts when its label lies in [0, K) and is not ignore_index.
 *   dva_csr_nll_fwd : loss[0] = mean over counted views of lse - x[label] (NaN when none counts), from
 *                     per-CTA fp64 partials (dva_csr_nll_fwd_workspace_bytes(N) bytes of workspace) summed in
 *                     a fixed order; lse [V] fp32 (nullable) = log-sum-exp of each row, for the backward;
 *                     stats [3] int64 = {counted views, views whose label is neither ignore_index nor in
 *                     [0, K), 1 if csr_idx does not run from 0 to V}.  Such labels and rows are never read
 *                     through; the caller raises on stats[1] / stats[2].
 *   dva_csr_nll_bwd : grad_logits [V, K] (logits' dtype) = grad_loss[0] / stats[0] * (exp(x - lse) - onehot),
 *                     0 on views that do not count; every element is written.
 *   Bytes: the forward reads the logits once, the backward reads them once and writes the gradient once. */
size_t dva_csr_nll_fwd_workspace_bytes(int64_t N);
int dva_csr_nll_fwd(const void* logits, int dtype, const int64_t* labels, const int64_t* csr_idx, int64_t V,
                    int64_t N, int K, int64_t ignore_index, float* lse, float* loss, int64_t* stats,
                    void* workspace, size_t workspace_bytes, void* stream);
int dva_csr_nll_bwd(const void* logits, int dtype, const int64_t* labels, const int64_t* csr_idx, int64_t V,
                    int64_t N, int K, int64_t ignore_index, const float* lse, const float* grad_loss,
                    const int64_t* stats, void* grad_logits, void* stream);

/* L2  class-weighted log-softmax NLL       replaces models/segmentation/sparseconv3d.py:41-58
 *   F.nll_loss(F.log_softmax(logits), labels, ignore_index=-1, weight=dataset.weight_classes), mean reduction,
 *   over the same inputs as L1 plus weight [K] float32 (device).  Separate kernels: L1 keeps its code and bits.
 *   dva_csr_nll_weighted_fwd : loss[0] = sum_v w[y_v] (lse_v - x_v[y_v]) / W with W = sum_v w[y_v] over the
 *                              counted views (fp64 per-CTA partials, dva_csr_nll_weighted_fwd_workspace_bytes(N)
 *                              bytes, summed in a fixed order; NaN when W is 0, as in torch); wsum[0] = W (fp64)
 *                              for the backward; lse and stats as L1.
 *   dva_csr_nll_weighted_bwd : grad_logits = grad_loss[0] / W * w[y_v] * (exp(x - lse) - onehot), 0 on views that
 *                              do not count.  With w = 1 both give L1's bits. */
size_t dva_csr_nll_weighted_fwd_workspace_bytes(int64_t N);
int dva_csr_nll_weighted_fwd(const void* logits, int dtype, const int64_t* labels, const int64_t* csr_idx, int64_t V,
                             int64_t N, int K, int64_t ignore_index, const float* weight, float* lse, float* loss,
                             double* wsum, int64_t* stats, void* workspace, size_t workspace_bytes, void* stream);
int dva_csr_nll_weighted_bwd(const void* logits, int dtype, const int64_t* labels, const int64_t* csr_idx, int64_t V,
                             int64_t N, int K, int64_t ignore_index, const float* weight, const float* lse,
                             const float* grad_loss, const double* wsum, void* grad_logits, void* stream);

/* L3  Lovász-softmax                        replaces metrics/lovasz_loss.py:155-230 (lovasz_softmax_flat after
 *                                           flatten_probas, per_image=False), called by
 *                                           models/segmentation/sparseconv3d.py:55-57 and
 *                                           models/segmentation/multimodal/sparseconv3d.py:163-181
 *   probas [P, K] (fp32 / bf16 / fp16 storage, fp32 math, 1 <= K <= 64), log-probabilities when log_probs (exp
 *   taken in the kernel), labels [P] int64; a point whose label is ignore_index is left out.
 *   dva_lovasz_keys : keys [K, P] fp32 = |fg - p| for valid points, -1 for ignored ones.  The caller sorts each
 *                     row descending and stable into sorted_keys [K, P] and perm [K, P] int64.
 *   dva_lovasz_fwd  : fgs [K, P] uint8 = fg in sorted order; gsorted [K, P] fp32 (nullable: no gradient) = the
 *                     Jaccard differences (lovasz_grad) in sorted order, 0 for ignored points; loss[0] = the mean
 *                     over kept classes of sum e_sorted g, kept_c = class_mult[c] (0 when present and class c
 *                     has no valid point), 0 when nothing is kept; scale [K] = kept_c / sum kept.  fp64
 *                     partials in a fixed order (dva_lovasz_fwd_workspace_bytes(P, K) bytes of workspace).
 *   dva_lovasz_bwd  : grad [P, K] (probas' dtype) = -sign(fg - p) g scale_c grad_loss[0], times p when log_probs,
 *                     0 for ignored points; every element written once through perm. */
int dva_lovasz_keys(const void* probas, int dtype, int log_probs, const int64_t* labels, int64_t P, int K,
                    int64_t ignore_index, float* keys, void* stream);
size_t dva_lovasz_fwd_workspace_bytes(int64_t P, int K);
int dva_lovasz_fwd(const float* sorted_keys, const int64_t* perm, const int64_t* labels, int64_t P, int K,
                   const int* class_mult, int present, uint8_t* fgs, float* gsorted, float* loss, float* scale,
                   void* workspace, size_t workspace_bytes, void* stream);
int dva_lovasz_bwd(const void* probas, int dtype, int log_probs, const float* sorted_keys, const int64_t* perm,
                   const uint8_t* fgs, const float* gsorted, const float* scale, const float* grad_loss, int64_t P,
                   int K, void* grad, void* stream);

/* C1  CSR pointers from sorted dense ids     replaces csr.py:158-172 + :197-229
 *   ids [n] int64 sorted ascending, values in [0,num_groups) -> ptr [num_groups+1] int64 with
 *   empty groups inserted (from_dense + insert_empty_groups, image.py:1787-1793). */
int dva_csr_pointers_from_sorted(const int64_t* ids, int64_t* ptr, int64_t n, int64_t num_groups,
                                 void* stream);

/* C1  value index of a group selection       replaces csr.py:235-264 (_index_select_pointers)
 *   ptr_new [k+1] must already hold the exclusive scan of the selected group sizes;
 *   val_idx[p] = ptr[sel[i]] + (p - ptr_new[i]) for p in [ptr_new[i], ptr_new[i+1]). */
int dva_csr_select_values(const int64_t* ptr, const int64_t* sel, const int64_t* ptr_new,
                          int64_t* val_idx, int64_t k, int64_t n_new_items, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DVA_B200_H_ */
