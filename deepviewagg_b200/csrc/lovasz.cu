// Lovász-softmax loss over [P, K] class probabilities (metrics/lovasz_loss.py:155-230, lovasz_softmax_flat
// after flatten_probas, per_image=False), all K classes at once instead of one sort / gather / cumsum / dot
// per class:
//
//   1. lovasz_keys_kernel: keys [K, P] fp32, keys[c, i] = |fg_ic - p_ic| (fg_ic = label_i == c) for a valid
//      point, -1 for an ignored one.  Errors are >= 0, so a descending sort puts every ignored point after
//      every valid point of its class; no compaction, no host sync.
//   2. the caller sorts each class row, descending and stable (torch.sort, CUB's segmented radix sort):
//      sorted keys and the permutation perm [K, P].
//   3. lovasz_fg_kernel (tiles of kLvTile sorted entries): fg in sorted order (uint8 [K, P]) and its count
//      per tile.  lovasz_loss_kernel: the tile's fg prefix from the tile counts, a block scan, then
//      Jaccard J_j = (j + 1) / (gts + j + 1 - F_j) (F_j = fg count up to sorted position j, gts = all fg of
//      the class; the reference's 1 - (gts - F_j) / (gts + (j + 1 - F_j))), g_j = J_j - J_{j-1} in fp64,
//      and the partial sum of e_j g_j (fp64).  An ignored entry has g = 0 and e = 0.
//      lovasz_finalize_kernel (one CTA): per-class sums in a fixed order, the mean over kept classes
//      (weights mult_c: 'all' / 'present' / a class list with repeats), and scale_c = kept_c / n_kept.
//   4. lovasz_bwd_kernel: grad[i, c] = -sign(fg - p) g_j scale_c upstream (times p with log_probs), written
//      through the permutation: every element once, no atomics; 0 for an ignored point.
//
// Ties: the loss does not depend on the order of equal errors, the gradient of one element of a tied
// block does; the stable sort breaks ties by point index.
#include "dva_common.cuh"

// namespace dva_loss: the loss kernels of the sparse-conv models (case table: tests/test_loss_matrix_table.py)
namespace dva_loss {
using namespace dva;

constexpr int kLvThreads = 256;
constexpr int kLvItems = 16;
constexpr int kLvTile = kLvThreads * kLvItems;
constexpr int kLvMaxK = 64;

static inline int lv_tiles(int64_t P) { return (int)((P + kLvTile - 1) / kLvTile); }

template <typename T, bool kLog>
__device__ __forceinline__ float lv_prob(const T* __restrict__ probas, int64_t i, int K, int c) {
  const float x = Cvt<T>::to_f(probas[i * K + c]);
  return kLog ? expf(x) : x;
}

template <typename T, bool kLog>
__global__ void __launch_bounds__(kLvThreads)
lovasz_keys_kernel(const T* __restrict__ probas, const int64_t* __restrict__ labels, int64_t P, int K,
                   int64_t ignore, float* __restrict__ keys) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t y = labels[i];
    const bool valid = y != ignore;
    for (int c = 0; c < K; ++c)
      keys[c * P + i] = valid ? fabsf((y == c ? 1.f : 0.f) - lv_prob<T, kLog>(probas, i, K, c)) : -1.f;
  }
}

// grid (tiles, K): fg of every sorted entry and the fg count of the tile
__global__ void __launch_bounds__(kLvThreads)
lovasz_fg_kernel(const float* __restrict__ skeys, const int64_t* __restrict__ perm,
                 const int64_t* __restrict__ labels, int64_t P, int ntiles, uint8_t* __restrict__ fgs,
                 int* __restrict__ tile_fg) {
  const int c = blockIdx.y;
  const int64_t base = (int64_t)c * P, t0 = (int64_t)blockIdx.x * kLvTile;
  int cnt = 0;
  for (int k = threadIdx.x; k < kLvTile; k += kLvThreads) {
    const int64_t j = t0 + k;
    if (j >= P) break;
    const bool fg = skeys[base + j] >= 0.f && labels[perm[base + j]] == c;
    fgs[base + j] = fg;
    cnt += fg;
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  __shared__ int sh[kLvThreads / 32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kLvThreads / 32; ++w) t += sh[w];
    tile_fg[c * ntiles + blockIdx.x] = t;
  }
}

// grid (tiles, K): Jaccard differences g of the tile (written when gsorted != NULL) and sum e g (fp64)
__global__ void __launch_bounds__(kLvThreads)
lovasz_loss_kernel(const float* __restrict__ skeys, const uint8_t* __restrict__ fgs, const int* __restrict__ tile_fg,
                   int64_t P, int ntiles, float* __restrict__ gsorted, double* __restrict__ part) {
  const int c = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = (int64_t)c * P, t0 = (int64_t)blockIdx.x * kLvTile;
  const int n = (int)min((int64_t)kLvTile, P - t0);
  __shared__ float sk[kLvTile];
  __shared__ uint8_t sf[kLvTile];
  __shared__ long long sred[2][kLvThreads / 32];
  __shared__ int sscan[kLvThreads / 32];
  __shared__ double sacc[kLvThreads / 32];

  // fg before this tile and in the whole class
  long long before = 0, gts = 0;
  for (int s = threadIdx.x; s < ntiles; s += kLvThreads) {
    const int v = tile_fg[c * ntiles + s];
    gts += v;
    if (s < (int)blockIdx.x) before += v;
  }
  for (int k = threadIdx.x; k < kLvTile; k += kLvThreads) {
    sk[k] = k < n ? skeys[base + t0 + k] : -1.f;
    sf[k] = k < n ? fgs[base + t0 + k] : 0;
  }
  for (int o = 16; o > 0; o >>= 1) {
    before += __shfl_down_sync(0xffffffffu, before, o);
    gts += __shfl_down_sync(0xffffffffu, gts, o);
  }
  if (lane == 0) { sred[0][warp] = before; sred[1][warp] = gts; }
  __syncthreads();
  before = gts = 0;
  for (int w = 0; w < kLvThreads / 32; ++w) { before += sred[0][w]; gts += sred[1][w]; }

  // block exclusive scan of the per-thread fg counts (kLvItems consecutive entries per thread)
  const int k0 = threadIdx.x * kLvItems;
  int mine = 0;
#pragma unroll
  for (int q = 0; q < kLvItems; ++q) mine += sf[k0 + q];
  int incl = mine;
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) sscan[warp] = incl;
  __syncthreads();
  int woff = 0;
  for (int w = 0; w < warp; ++w) woff += sscan[w];
  long long F = before + woff + incl - mine;   // fg count before this thread's first entry

  const double dg = (double)gts;
  double acc = 0.0;
#pragma unroll 4
  for (int q = 0; q < kLvItems; ++q) {
    const int k = k0 + q;
    const float e = sk[k];
    float gf = 0.f;
    if (e >= 0.f) {                               // a valid entry (ignored ones and the tile's tail are -1)
      const long long j = t0 + k;
      const long long Fp = F;                     // fg count before position j
      F += sf[k];
      const double Jj = (double)(j + 1) / (dg + (double)(j + 1 - F));
      const double Jp = j == 0 ? 0.0 : (double)j / (dg + (double)(j - Fp));
      const double g = Jj - Jp;
      acc += (double)e * g;
      gf = (float)g;
    }
    sk[k] = gf;                                   // this thread's own entries: no race with other threads
  }
  __syncthreads();
  if (gsorted)
    for (int k = threadIdx.x; k < n; k += kLvThreads) gsorted[base + t0 + k] = sk[k];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if (lane == 0) sacc[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kLvThreads / 32; ++w) t += sacc[w];
    part[c * ntiles + blockIdx.x] = t;
  }
}

// one CTA: per-class loss and fg count (warp w sums the tiles of classes w, w + 8, ... in a fixed order),
// then the mean over kept classes; 0 when no class is kept
__global__ void __launch_bounds__(kLvThreads)
lovasz_finalize_kernel(const double* __restrict__ part, const int* __restrict__ tile_fg, int ntiles, int K,
                       const int* __restrict__ mult, int present, float* __restrict__ loss,
                       float* __restrict__ scale) {
  __shared__ double sl[kLvMaxK];
  __shared__ long long sg[kLvMaxK];
  __shared__ double skept[kLvMaxK];
  __shared__ double sn;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = warp; c < K; c += kLvThreads / 32) {
    double a = 0.0;
    long long g = 0;
    for (int s = lane; s < ntiles; s += 32) { a += part[c * ntiles + s]; g += tile_fg[c * ntiles + s]; }
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_down_sync(0xffffffffu, a, o);
      g += __shfl_down_sync(0xffffffffu, g, o);
    }
    if (lane == 0) { sl[c] = a; sg[c] = g; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sum = 0.0, nk = 0.0;
    for (int c = 0; c < K; ++c) {
      const double kept = (present && sg[c] == 0) ? 0.0 : (double)mult[c];
      skept[c] = kept;
      sum += kept * sl[c];
      nk += kept;
    }
    loss[0] = nk > 0.0 ? (float)(sum / nk) : 0.f;
    sn = nk;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < K; c += kLvThreads) scale[c] = sn > 0.0 ? (float)(skept[c] / sn) : 0.f;
}

template <typename T, bool kLog>
__global__ void __launch_bounds__(kLvThreads)
lovasz_bwd_kernel(const T* __restrict__ probas, const float* __restrict__ skeys, const int64_t* __restrict__ perm,
                  const uint8_t* __restrict__ fgs, const float* __restrict__ gsorted, const float* __restrict__ scale,
                  const float* __restrict__ grad_loss, int64_t P, int K, T* __restrict__ grad) {
  const int c = blockIdx.y;
  const int64_t base = (int64_t)c * P;
  const float s = scale[c] * grad_loss[0];
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < P; j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = perm[base + j];
    float v = 0.f;
    if (skeys[base + j] >= 0.f) {
      const float p = lv_prob<T, kLog>(probas, i, K, c);
      const float d = (fgs[base + j] ? 1.f : 0.f) - p;
      const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);   // d|fg - p| / dp = -sign(fg - p)
      v = -sg * gsorted[base + j] * s;
      if (kLog) v *= p;
    }
    grad[i * K + c] = Cvt<T>::from_f(v);
  }
}

template <typename F> bool with_log(int log_probs, F&& f) {
  if (log_probs) f(std::true_type{}); else f(std::false_type{});
  return true;
}

}  // namespace dva_loss

using namespace dva;
using namespace dva_loss;

extern "C" int dva_lovasz_keys(const void* probas, int dtype, int log_probs, const int64_t* labels, int64_t P, int K,
                               int64_t ignore_index, float* keys, void* stream) {
  if (P < 0 || K < 1) return fail(DVA_EINVAL, "lovasz_keys: bad sizes");
  if (K > kLvMaxK) return fail(DVA_EUNSUPPORTED, "lovasz_keys: K must be in [1, 64]");
  if (P == 0) return DVA_OK;
  if (!probas || !labels || !keys) return fail(DVA_EINVAL, "lovasz_keys: null pointer");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "lovasz_keys: unknown dtype");
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    with_log(log_probs, [&](auto lg) {
      lovasz_keys_kernel<T, decltype(lg)::value><<<grid_cap(P, kLvThreads, 8), kLvThreads, 0, (cudaStream_t)stream>>>(
          (const T*)probas, labels, P, K, ignore_index, keys);
    });
  });
  return check_launch("lovasz_keys");
}

extern "C" size_t dva_lovasz_fwd_workspace_bytes(int64_t P, int K) {
  const size_t n = (size_t)lv_tiles(P) * (size_t)(K > 0 ? K : 0);
  return round256(n * sizeof(double)) + n * sizeof(int);
}

extern "C" int dva_lovasz_fwd(const float* sorted_keys, const int64_t* perm, const int64_t* labels, int64_t P, int K,
                              const int* class_mult, int present, uint8_t* fgs, float* gsorted, float* loss,
                              float* scale, void* workspace, size_t workspace_bytes, void* stream) {
  if (P < 0 || K < 1) return fail(DVA_EINVAL, "lovasz_fwd: bad sizes");
  if (K > kLvMaxK) return fail(DVA_EUNSUPPORTED, "lovasz_fwd: K must be in [1, 64]");
  if (P >= (int64_t)INT32_MAX * kLvTile / kLvMaxK) return fail(DVA_EUNSUPPORTED, "lovasz_fwd: too many points");
  if (!class_mult || !loss || !scale || !workspace || (P > 0 && (!sorted_keys || !perm || !labels || !fgs)))
    return fail(DVA_EINVAL, "lovasz_fwd: null pointer");
  if (workspace_bytes < dva_lovasz_fwd_workspace_bytes(P, K)) return fail(DVA_EINVAL, "lovasz_fwd: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int nt = lv_tiles(P);
  double* part = (double*)workspace;
  int* tile_fg = (int*)((uint8_t*)workspace + round256((size_t)nt * K * sizeof(double)));
  if (nt > 0) {
    const dim3 grid(nt, K);
    lovasz_fg_kernel<<<grid, kLvThreads, 0, st>>>(sorted_keys, perm, labels, P, nt, fgs, tile_fg);
    int rc = check_launch("lovasz_fg");
    if (rc != DVA_OK) return rc;
    lovasz_loss_kernel<<<grid, kLvThreads, 0, st>>>(sorted_keys, fgs, tile_fg, P, nt, gsorted, part);
    rc = check_launch("lovasz_loss");
    if (rc != DVA_OK) return rc;
  }
  lovasz_finalize_kernel<<<1, kLvThreads, 0, st>>>(part, tile_fg, nt, K, class_mult, present, loss, scale);
  return check_launch("lovasz_finalize");
}

extern "C" int dva_lovasz_bwd(const void* probas, int dtype, int log_probs, const float* sorted_keys,
                              const int64_t* perm, const uint8_t* fgs, const float* gsorted, const float* scale,
                              const float* grad_loss, int64_t P, int K, void* grad, void* stream) {
  if (P < 0 || K < 1) return fail(DVA_EINVAL, "lovasz_bwd: bad sizes");
  if (K > kLvMaxK) return fail(DVA_EUNSUPPORTED, "lovasz_bwd: K must be in [1, 64]");
  if (P == 0) return DVA_OK;
  if (!probas || !sorted_keys || !perm || !fgs || !gsorted || !scale || !grad_loss || !grad)
    return fail(DVA_EINVAL, "lovasz_bwd: null pointer");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "lovasz_bwd: unknown dtype");
  const dim3 grid((unsigned)grid_cap(P, kLvThreads, 8), K);
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    with_log(log_probs, [&](auto lg) {
      lovasz_bwd_kernel<T, decltype(lg)::value><<<grid, kLvThreads, 0, (cudaStream_t)stream>>>(
          (const T*)probas, sorted_keys, perm, fgs, gsorted, scale, grad_loss, P, K, (T*)grad);
    });
  });
  return check_launch("lovasz_bwd");
}
