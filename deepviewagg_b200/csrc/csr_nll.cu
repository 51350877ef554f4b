// Log-softmax NLL over a view CSR (models/segmentation/multimodal/no3d.py:144-154):
//
//   nll_loss(log_softmax(logits), repeat_interleave(labels, counts), ignore_index)   (mean)
//
// without the [V] int64 target tensor and the [V, K] log-prob tensor the reference materialises.
// One thread per point walks the rows of its views (csr_idx == NULL: one view per point); the
// target of a view is its point's label.  A row is read once: an online max / sum gives
// lse = log(sum exp(x)) and the row loss is (m - x[y]) + log(s), all in fp32.
//
// Forward: per-CTA partial sums (fp64 loss, int64 counts) written to the workspace, combined by a
// one-CTA kernel in a fixed order: the result does not depend on scheduling.  Labels that are
// neither ignore_index nor in [0, K) are counted (never read through) and reported in stats[1];
// a csr_idx that does not run from 0 to V is reported in stats[2] (rows past V are never read).
// Backward: grad = g / count * (exp(x - lse) - onehot), zeros for ignored views; lse [V] is the
// forward's, so the backward reads each row once and writes it once.
#include "dva_common.cuh"

namespace dva {

constexpr int kNllThreads = 256;
constexpr int kNllMaxK = 64;

// one forward partial per CTA: the workspace query and the launches share the grid
static inline int nll_blocks(int64_t N) { return grid_cap(N, kNllThreads, 8); }

struct NllPartial {
  double loss;
  long long count, bad;
};

template <typename T>
__global__ void __launch_bounds__(kNllThreads)
csr_nll_fwd_kernel(const T* __restrict__ logits, const int64_t* __restrict__ labels,
                   const int64_t* __restrict__ csr, int64_t V, int64_t N, int K, int64_t ignore,
                   float* __restrict__ lse, NllPartial* __restrict__ part) {
  double acc = 0.0;
  long long cnt = 0, bad = 0;
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < N; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t y = labels[p];
    int64_t v0 = csr ? csr[p] : p, v1 = csr ? csr[p + 1] : p + 1;
    v0 = min(max(v0, (int64_t)0), V);
    v1 = min(max(v1, v0), V);
    const bool valid = y >= 0 && y < K && y != ignore;
    if (!valid && y != ignore) bad += v1 - v0;
    for (int64_t v = v0; v < v1; ++v) {
      const T* __restrict__ row = logits + v * K;
      float m = -INFINITY, s = 0.f, xy = 0.f;
      for (int j = 0; j < K; ++j) {
        const float x = Cvt<T>::to_f(row[j]);
        // a -inf logit adds exp(-inf) = 0; skipping it keeps exp(-inf - -inf) = NaN out of s while m is
        // still -inf, so a row with one finite logit has a finite lse (a row of -inf only stays NaN, as in torch)
        if (x > m) { s = s * expf(m - x) + 1.f; m = x; }
        else if (x != -INFINITY) s += expf(x - m);
        if (j == y) xy = x;
      }
      const float ls = logf(s);
      if (lse) lse[v] = m + ls;
      if (valid) { acc += (double)((m - xy) + ls); ++cnt; }
    }
  }
  // fixed-order block reduction
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_down_sync(0xffffffffu, acc, o);
    cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    bad += __shfl_down_sync(0xffffffffu, bad, o);
  }
  __shared__ NllPartial sh[kNllThreads / 32];
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) sh[w] = NllPartial{acc, cnt, bad};
  __syncthreads();
  if (threadIdx.x == 0) {
    NllPartial t{0.0, 0, 0};
    for (int i = 0; i < kNllThreads / 32; ++i) { t.loss += sh[i].loss; t.count += sh[i].count; t.bad += sh[i].bad; }
    part[blockIdx.x] = t;
  }
}

// one CTA: partials in a fixed order -> loss = sum / count (NaN when nothing counts), stats
__global__ void __launch_bounds__(kNllThreads)
csr_nll_finalize_kernel(const NllPartial* __restrict__ part, int nparts, const int64_t* __restrict__ csr,
                        int64_t V, int64_t N, float* __restrict__ loss, int64_t* __restrict__ stats) {
  double acc = 0.0;
  long long cnt = 0, bad = 0;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) { acc += part[i].loss; cnt += part[i].count; bad += part[i].bad; }
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_down_sync(0xffffffffu, acc, o);
    cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    bad += __shfl_down_sync(0xffffffffu, bad, o);
  }
  __shared__ NllPartial sh[kNllThreads / 32];
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) sh[w] = NllPartial{acc, cnt, bad};
  __syncthreads();
  if (threadIdx.x == 0) {
    NllPartial t{0.0, 0, 0};
    for (int i = 0; i < kNllThreads / 32; ++i) { t.loss += sh[i].loss; t.count += sh[i].count; t.bad += sh[i].bad; }
    loss[0] = (float)(t.loss / (double)t.count);          // 0 / 0 = NaN, as F.nll_loss over no element
    stats[0] = t.count;
    stats[1] = t.bad;
    stats[2] = (csr != nullptr && (csr[0] != 0 || csr[N] != V)) ? 1 : 0;
  }
}

template <typename T>
__global__ void __launch_bounds__(kNllThreads)
csr_nll_bwd_kernel(const T* __restrict__ logits, const int64_t* __restrict__ labels,
                   const int64_t* __restrict__ csr, int64_t V, int64_t N, int K, int64_t ignore,
                   const float* __restrict__ lse, const float* __restrict__ grad_loss,
                   const int64_t* __restrict__ stats, T* __restrict__ grad) {
  const float scale = (float)((double)grad_loss[0] / (double)stats[0]);
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < N; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t y = labels[p];
    int64_t v0 = csr ? csr[p] : p, v1 = csr ? csr[p + 1] : p + 1;
    v0 = min(max(v0, (int64_t)0), V);
    v1 = min(max(v1, v0), V);
    const bool valid = y >= 0 && y < K && y != ignore;
    for (int64_t v = v0; v < v1; ++v) {
      const T* __restrict__ row = logits + v * K;
      T* __restrict__ g = grad + v * K;
      if (!valid) {
        for (int j = 0; j < K; ++j) g[j] = Cvt<T>::from_f(0.f);
        continue;
      }
      const float l = lse[v];
      for (int j = 0; j < K; ++j) {
        const float sm = expf(Cvt<T>::to_f(row[j]) - l);
        g[j] = Cvt<T>::from_f(scale * (j == y ? sm - 1.f : sm));
      }
    }
  }
}

}  // namespace dva

using namespace dva;

extern "C" size_t dva_csr_nll_fwd_workspace_bytes(int64_t N) {
  return (size_t)nll_blocks(N) * sizeof(NllPartial);
}

extern "C" int dva_csr_nll_fwd(const void* logits, int dtype, const int64_t* labels, const int64_t* csr_idx,
                               int64_t V, int64_t N, int K, int64_t ignore_index, float* lse, float* loss,
                               int64_t* stats, void* workspace, size_t workspace_bytes, void* stream) {
  if (V < 0 || N < 0 || K < 1) return fail(DVA_EINVAL, "csr_nll_fwd: bad sizes");
  if (K > kNllMaxK) return fail(DVA_EUNSUPPORTED, "csr_nll_fwd: K must be in [1, 64]");
  if (csr_idx == nullptr && V != N) return fail(DVA_EINVAL, "csr_nll_fwd: without csr_idx, V must equal N");
  if (!loss || !stats || !workspace || (N > 0 && !labels) || (V > 0 && !logits))
    return fail(DVA_EINVAL, "csr_nll_fwd: null pointer");
  const int nb = N > 0 ? nll_blocks(N) : 0;
  if (workspace_bytes < (size_t)nb * sizeof(NllPartial)) return fail(DVA_EINVAL, "csr_nll_fwd: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  NllPartial* part = (NllPartial*)workspace;
  if (nb > 0) {
    if (!known_dtype(dtype)) return fail(DVA_EINVAL, "csr_nll_fwd: unknown dtype");
    with_dtype(dtype, [&](auto t) {
      using T = decltype(t);
      csr_nll_fwd_kernel<T><<<nb, kNllThreads, 0, st>>>((const T*)logits, labels, csr_idx, V, N, K, ignore_index,
                                                         lse, part);
    });
    const int rc = check_launch("csr_nll_fwd");
    if (rc != DVA_OK) return rc;
  }
  csr_nll_finalize_kernel<<<1, kNllThreads, 0, st>>>(part, nb, csr_idx, V, N, loss, stats);
  return check_launch("csr_nll_finalize");
}

extern "C" int dva_csr_nll_bwd(const void* logits, int dtype, const int64_t* labels, const int64_t* csr_idx,
                               int64_t V, int64_t N, int K, int64_t ignore_index, const float* lse,
                               const float* grad_loss, const int64_t* stats, void* grad_logits, void* stream) {
  if (V < 0 || N < 0 || K < 1) return fail(DVA_EINVAL, "csr_nll_bwd: bad sizes");
  if (K > kNllMaxK) return fail(DVA_EUNSUPPORTED, "csr_nll_bwd: K must be in [1, 64]");
  if (csr_idx == nullptr && V != N) return fail(DVA_EINVAL, "csr_nll_bwd: without csr_idx, V must equal N");
  if (V == 0 || N == 0) return DVA_OK;
  if (!logits || !labels || !lse || !grad_loss || !stats || !grad_logits) return fail(DVA_EINVAL, "csr_nll_bwd: null pointer");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "csr_nll_bwd: unknown dtype");
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    csr_nll_bwd_kernel<T><<<nll_blocks(N), kNllThreads, 0, (cudaStream_t)stream>>>(
        (const T*)logits, labels, csr_idx, V, N, K, ignore_index, lse, grad_loss, stats, (T*)grad_logits);
  });
  return check_launch("csr_nll_bwd");
}
