// Fused BatchNorm1d (+ LeakyReLU) over the rows of a [R, C] activation matrix: the second half of
// every MLP layer of the pools (reference core/common_modules/base_modules.py:38-48:
// Linear(bias=False) -> FastBatchNorm1d -> LeakyReLU(0.2), :131-156 FastBatchNorm1d).
//
// The reference runs, per layer, GEMM | BN statistics | BN transform | in-place LeakyReLU (and the
// mirrored chain backward) = 6 passes over [R,C] forward.  Here: one statistics pass (read z) and
// one apply pass (read z, write y) forward; one reduce pass (read dy, z) and one apply pass (read
// dy, z, write dz) backward.  All four kernels are HBM-bound streams; per-column sums are
// deterministic (per-CTA partials + a fixed-order second stage in fp64).
//
// Layout: z row-major [R, C].  A CTA of 256 threads covers a slab of rows; thread t owns column
// group (t % TC) of VEC consecutive columns and walks rows (t / TC), (t / TC) + RG, ... so every
// warp-level access is a run of consecutive addresses.
// Variance uses sums shifted by the column's first-row value (no catastrophic cancellation).
#include "dva_common.cuh"

namespace dva {

constexpr int kBnThreads = 256;

template <typename T, int VEC>
__device__ __forceinline__ void ld_vec(const T* p, float (&f)[VEC]) {
  if constexpr (VEC == 1) { f[0] = Cvt<T>::to_f(*p); }
  else { unpack16<T, VEC>(*reinterpret_cast<const uint4*>(p), f); }
}
template <typename T, int VEC>
__device__ __forceinline__ void st_vec(T* p, const float (&f)[VEC]) {
  if constexpr (VEC == 1) { *p = Cvt<T>::from_f(f[0]); }
  else { *reinterpret_cast<uint4*>(p) = pack16<T, VEC>(f); }
}

// ---- pass 1 (fwd): per-CTA partial sums of (z - shift) and (z - shift)^2 ------------------------
// partial [grid][2][C] fp32.  CV = C / VEC column groups; threads beyond the last full row group idle.
template <typename T, int VEC>
__global__ void __launch_bounds__(kBnThreads)
bn_stats_kernel(const T* __restrict__ z, float* __restrict__ partial, int64_t R, int C) {
  extern __shared__ float sm[];                       // [RG][2][CV*VEC]
  const int CV = C / VEC;
  const int TC = CV < kBnThreads ? CV : kBnThreads;   // threads across columns
  const int RG = kBnThreads / TC;                     // row groups per CTA
  const int tc = threadIdx.x % TC, rg = threadIdx.x / TC;
  const int64_t rows_per_cta = (R + gridDim.x - 1) / gridDim.x;
  const int64_t r0 = blockIdx.x * rows_per_cta, r1 = min(R, r0 + rows_per_cta);
  for (int cv = tc; cv < CV; cv += TC) {
    float s[VEC], q[VEC], sh[VEC];
    ld_vec<T, VEC>(z + cv * VEC, sh);                 // shift = row 0 (same for every CTA)
#pragma unroll
    for (int j = 0; j < VEC; ++j) { s[j] = 0.f; q[j] = 0.f; }
    if (rg < RG) {
      for (int64_t r = r0 + rg; r < r1; r += RG) {
        float v[VEC];
        ld_vec<T, VEC>(z + r * C + cv * VEC, v);
#pragma unroll
        for (int j = 0; j < VEC; ++j) { const float d = v[j] - sh[j]; s[j] += d; q[j] = fmaf(d, d, q[j]); }
      }
    }
    if (rg < RG) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        sm[(rg * 2 + 0) * C + cv * VEC + j] = s[j];
        sm[(rg * 2 + 1) * C + cv * VEC + j] = q[j];
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += kBnThreads) {
    const int which = c / C, col = c - which * C;
    float acc = 0.f;
    for (int g = 0; g < RG; ++g) acc += sm[(g * 2 + which) * C + col];
    partial[(int64_t)blockIdx.x * 2 * C + c] = acc;
  }
}

// ---- finalize (fwd): mean / invstd, running statistics (momentum, unbiased variance) --------------
// one warp per column: lanes stride over the CTA partials (fixed order -> deterministic), fp64 combine
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__global__ void __launch_bounds__(256)
bn_finalize_kernel(const T* __restrict__ z, const float* __restrict__ partial, int grid,
                   int64_t R, int C, float eps, float momentum, float* __restrict__ mean,
                   float* __restrict__ invstd, float* __restrict__ running_mean,
                   float* __restrict__ running_var) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  double s = 0.0, q = 0.0;
  for (int b = lane; b < grid; b += 32) {
    s += (double)partial[(int64_t)b * 2 * C + c];
    q += (double)partial[(int64_t)b * 2 * C + C + c];
  }
  s = warp_sum_d(s); q = warp_sum_d(q);
  if (lane != 0) return;
  const double n = (double)R, shift = (double)Cvt<T>::to_f(z[c]);
  const double ms = s / n;
  double var = q / n - ms * ms;
  if (var < 0.0) var = 0.0;
  const double mu = shift + ms;
  mean[c] = (float)mu;
  invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean != nullptr) {
    const double unbiased = R > 1 ? var * n / (n - 1.0) : var;
    running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * mu);
    running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unbiased);
  }
}

// ---- pass 2 (fwd): y = act(gamma * (z - mean) * invstd + beta) -------------------------------------
template <typename T, int VEC>
__global__ void __launch_bounds__(kBnThreads)
bn_apply_kernel(const T* __restrict__ z, const float* __restrict__ mean, const float* __restrict__ invstd,
                const float* __restrict__ gamma, const float* __restrict__ beta, T* __restrict__ y,
                int64_t R, int C, float slope) {
  // thread -> fixed column group (scale/shift in registers), rows strided over the whole grid
  const int CV = C / VEC;
  const int TC = CV < kBnThreads ? CV : kBnThreads;
  const int RG = kBnThreads / TC;
  const int tc = threadIdx.x % TC, rg = threadIdx.x / TC;
  if (rg >= RG) return;
  for (int cv = tc; cv < CV; cv += TC) {
    float sc[VEC], sh[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const int c = cv * VEC + j;
      sc[j] = (gamma ? gamma[c] : 1.f) * invstd[c];
      sh[j] = (beta ? beta[c] : 0.f) - mean[c] * sc[j];
    }
    const T* zp = z + cv * VEC;
    T* yp = y + cv * VEC;
    for (int64_t r = (int64_t)blockIdx.x * RG + rg; r < R; r += (int64_t)gridDim.x * RG) {
      float v[VEC];
      ld_vec<T, VEC>(zp + r * C, v);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float a = fmaf(v[j], sc[j], sh[j]);
        v[j] = a > 0.f ? a : a * slope;
      }
      st_vec<T, VEC>(yp + r * C, v);
    }
  }
}

// ---- pass 1 (bwd): per-CTA partials of sum(g) and sum(g * zhat), g = dy * act'(pre-activation) ----
template <typename T, int VEC>
__global__ void __launch_bounds__(kBnThreads)
bn_bwd_reduce_kernel(const T* __restrict__ dy, const T* __restrict__ z, const float* __restrict__ mean,
                     const float* __restrict__ invstd, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float* __restrict__ partial, int64_t R, int C,
                     float slope) {
  extern __shared__ float sm[];
  const int CV = C / VEC;
  const int TC = CV < kBnThreads ? CV : kBnThreads;
  const int RG = kBnThreads / TC;
  const int tc = threadIdx.x % TC, rg = threadIdx.x / TC;
  const int64_t rows_per_cta = (R + gridDim.x - 1) / gridDim.x;
  const int64_t r0 = blockIdx.x * rows_per_cta, r1 = min(R, r0 + rows_per_cta);
  for (int cv = tc; cv < CV; cv += TC) {
    float s[VEC], q[VEC], mu[VEC], is[VEC], sc[VEC], sh[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const int c = cv * VEC + j;
      s[j] = 0.f; q[j] = 0.f; mu[j] = mean[c]; is[j] = invstd[c];
      sc[j] = (gamma ? gamma[c] : 1.f) * is[j];
      sh[j] = (beta ? beta[c] : 0.f) - mu[j] * sc[j];
    }
    if (rg < RG) {
      for (int64_t r = r0 + rg; r < r1; r += RG) {
        float v[VEC], g[VEC];
        ld_vec<T, VEC>(z + r * C + cv * VEC, v);
        ld_vec<T, VEC>(dy + r * C + cv * VEC, g);
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          const float zh = (v[j] - mu[j]) * is[j];
          const float a = fmaf(v[j], sc[j], sh[j]);      // same expression as the forward: same sign
          const float gg = a > 0.f ? g[j] : g[j] * slope;
          s[j] += gg; q[j] = fmaf(gg, zh, q[j]);
        }
      }
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        sm[(rg * 2 + 0) * C + cv * VEC + j] = s[j];
        sm[(rg * 2 + 1) * C + cv * VEC + j] = q[j];
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += kBnThreads) {
    const int which = c / C, col = c - which * C;
    float acc = 0.f;
    for (int g = 0; g < RG; ++g) acc += sm[(g * 2 + which) * C + col];
    partial[(int64_t)blockIdx.x * 2 * C + c] = acc;
  }
}

// sums[0][c] = sum g (= d beta), sums[1][c] = sum g*zhat (= d gamma)
__global__ void __launch_bounds__(256)
bn_bwd_finalize_kernel(const float* __restrict__ partial, int grid, int C, float* __restrict__ sums) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= 2 * C) return;
  double acc = 0.0;
  for (int b = lane; b < grid; b += 32) acc += (double)partial[(int64_t)b * 2 * C + c];
  acc = warp_sum_d(acc);
  if (lane == 0) sums[c] = (float)acc;
}

// ---- pass 2 (bwd): dz = gamma*invstd * (g - mean(g) - zhat * mean(g*zhat))   [train]
//                    dz = gamma*invstd * g                                      [eval: fixed statistics]
template <typename T, int VEC>
__global__ void __launch_bounds__(kBnThreads)
bn_bwd_apply_kernel(const T* __restrict__ dy, const T* __restrict__ z, const float* __restrict__ mean,
                    const float* __restrict__ invstd, const float* __restrict__ gamma,
                    const float* __restrict__ beta, const float* __restrict__ sums, T* __restrict__ dz,
                    int64_t R, int C, float slope, int training) {
  const int CV = C / VEC;
  const int TC = CV < kBnThreads ? CV : kBnThreads;
  const int RG = kBnThreads / TC;
  const int tc = threadIdx.x % TC, rg = threadIdx.x / TC;
  if (rg >= RG) return;
  const float inv_n = 1.f / (float)R;
  for (int cv = tc; cv < CV; cv += TC) {
    float mu[VEC], is[VEC], sc[VEC], sh[VEC], k0[VEC], k1[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const int c = cv * VEC + j;
      mu[j] = mean[c]; is[j] = invstd[c];
      sc[j] = (gamma ? gamma[c] : 1.f) * is[j];
      sh[j] = (beta ? beta[c] : 0.f) - mu[j] * sc[j];
      k0[j] = training ? sums[c] * inv_n : 0.f;        // mean(g)
      k1[j] = training ? sums[C + c] * inv_n : 0.f;    // mean(g * zhat)
    }
    const T* zp = z + cv * VEC;
    const T* gp = dy + cv * VEC;
    T* op = dz + cv * VEC;
    for (int64_t r = (int64_t)blockIdx.x * RG + rg; r < R; r += (int64_t)gridDim.x * RG) {
      float v[VEC], g[VEC];
      ld_vec<T, VEC>(zp + r * C, v);
      ld_vec<T, VEC>(gp + r * C, g);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float a = fmaf(v[j], sc[j], sh[j]);
        const float gg = a > 0.f ? g[j] : g[j] * slope;
        const float zh = (v[j] - mu[j]) * is[j];
        v[j] = sc[j] * (gg - k0[j] - zh * k1[j]);
      }
      st_vec<T, VEC>(op + r * C, v);
    }
  }
}

// the reductions: at least 64 rows per CTA, 4 CTAs per SM
static int bn_grid_reduce(int64_t R) { return grid_cap(R, 64, 4); }
// rows per CTA of the streaming kernels (RG row groups of TC column threads)
static int bn_row_groups(int C, int vec) {
  const int CV = C / vec;
  return kBnThreads / (CV < kBnThreads ? CV : kBnThreads);
}
static size_t bn_smem(int C, int vec) { return (size_t)bn_row_groups(C, vec) * 2 * C * sizeof(float); }

}  // namespace dva

using namespace dva;

extern "C" size_t dva_bn_workspace_bytes(int64_t R, int64_t C) {
  return (size_t)bn_grid_reduce(R) * 2 * (size_t)(C > 0 ? C : 1) * sizeof(float);
}

// statistics pass (reduce) and row pass (stream) of one dtype and vector width
template <typename T, int VEC>
static int bn_fwd_launch(const void* z, const float* gamma, const float* beta, float* running_mean, float* running_var,
                         float* mean, float* invstd, void* y, int64_t R, int C, float eps, float momentum, float slope,
                         int training, void* workspace, cudaStream_t st) {
  int rc;
  if (training) {
    const int grid = bn_grid_reduce(R);
    const size_t smem = bn_smem(C, VEC);
    (void)smem_opt_in(bn_stats_kernel<T, VEC>, smem);
    bn_stats_kernel<T, VEC><<<grid, kBnThreads, smem, st>>>((const T*)z, (float*)workspace, R, C);
    if ((rc = check_launch("bn_stats"))) return rc;
    bn_finalize_kernel<T><<<(C + 7) / 8, 256, 0, st>>>((const T*)z, (const float*)workspace, grid, R, C, eps, momentum,
                                                       mean, invstd, running_mean, running_var);
    if ((rc = check_launch("bn_finalize"))) return rc;
  }
  // eval: fixed statistics, mean = running_mean, invstd = rsqrt(running_var + eps) computed by the host mirror
  bn_apply_kernel<T, VEC><<<grid_cap(R, bn_row_groups(C, VEC), 8), kBnThreads, 0, st>>>(
      (const T*)z, mean, invstd, gamma, beta, (T*)y, R, C, slope);
  return check_launch("bn_apply");
}

template <typename T, int VEC>
static int bn_bwd_launch(const void* dy, const void* z, const float* gamma, const float* beta, const float* mean,
                         const float* invstd, void* dz, float* dgamma_dbeta, int64_t R, int C, float slope, int training,
                         void* workspace, cudaStream_t st) {
  const int grid = bn_grid_reduce(R);
  const size_t smem = bn_smem(C, VEC);
  (void)smem_opt_in(bn_bwd_reduce_kernel<T, VEC>, smem);
  bn_bwd_reduce_kernel<T, VEC><<<grid, kBnThreads, smem, st>>>((const T*)dy, (const T*)z, mean, invstd, gamma, beta,
                                                             (float*)workspace, R, C, slope);
  int rc;
  if ((rc = check_launch("bn_bwd_reduce"))) return rc;
  // dgamma_dbeta = [sum g ; sum g*zhat]  (note the order: [0] = d beta, [1] = d gamma)
  bn_bwd_finalize_kernel<<<(2 * C + 7) / 8, 256, 0, st>>>((const float*)workspace, grid, C, dgamma_dbeta);
  if ((rc = check_launch("bn_bwd_finalize"))) return rc;
  if (!dz) return DVA_OK;
  bn_bwd_apply_kernel<T, VEC><<<grid_cap(R, bn_row_groups(C, VEC), 8), kBnThreads, 0, st>>>(
      (const T*)dy, (const T*)z, mean, invstd, gamma, beta, dgamma_dbeta, (T*)dz, R, C, slope, training);
  return check_launch("bn_bwd_apply");
}

extern "C" int dva_bn_act_fwd(const void* z, const float* gamma, const float* beta, float* running_mean,
                              float* running_var, float* mean, float* invstd, void* y, int64_t R, int64_t C,
                              float eps, float momentum, float slope, int training, int dtype,
                              void* workspace, size_t workspace_bytes, void* stream) {
  if (R < 0 || C < 1 || C > 65536) return fail(DVA_EINVAL, "bn_act_fwd: bad sizes");
  if (R == 0) return DVA_OK;
  if (!z || !y || !mean || !invstd) return fail(DVA_EINVAL, "bn_act_fwd: null pointer");
  if (training && (!workspace || workspace_bytes < dva_bn_workspace_bytes(R, C)))
    return fail(DVA_EINVAL, "bn_act_fwd: workspace too small");
  if (!training && (!running_mean || !running_var)) return fail(DVA_EINVAL, "bn_act_fwd: eval mode needs running statistics");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "bn_act_fwd: unknown dtype");
  cudaStream_t st = (cudaStream_t)stream;
  return with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    const bool vec = vec16_ok<T>(C, z, y);
    if (training && bn_smem((int)C, vec ? Vec16<T>::N : 1) > 200 * 1024)
      return fail(DVA_EUNSUPPORTED, "bn_act_fwd: C too large for the reduction tile");
    auto launch = vec ? bn_fwd_launch<T, Vec16<T>::N> : bn_fwd_launch<T, 1>;
    return launch(z, gamma, beta, running_mean, running_var, mean, invstd, y, R, (int)C, eps, momentum, slope, training,
                  workspace, st);
  });
}

extern "C" int dva_bn_act_bwd(const void* dy, const void* z, const float* gamma, const float* beta,
                              const float* mean, const float* invstd, void* dz, float* dgamma_dbeta,
                              int64_t R, int64_t C, float slope, int training, int dtype, void* workspace,
                              size_t workspace_bytes, void* stream) {
  if (R < 0 || C < 1 || C > 65536) return fail(DVA_EINVAL, "bn_act_bwd: bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  if (R == 0) {
    if (dgamma_dbeta) cudaMemsetAsync(dgamma_dbeta, 0, 2 * C * sizeof(float), st);
    return DVA_OK;
  }
  // dz == nullptr: statistics pass only (the caller differentiates the rows itself: mlp_layer.cu)
  if (!dy || !z || !mean || !invstd || !dgamma_dbeta) return fail(DVA_EINVAL, "bn_act_bwd: null pointer");
  if (!workspace || workspace_bytes < dva_bn_workspace_bytes(R, C)) return fail(DVA_EINVAL, "bn_act_bwd: workspace too small");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "bn_act_bwd: unknown dtype");
  return with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    const bool vec = vec16_ok<T>(C, z, dy, dz);
    if (bn_smem((int)C, vec ? Vec16<T>::N : 1) > 200 * 1024)
      return fail(DVA_EUNSUPPORTED, "bn_act_bwd: C too large for the reduction tile");
    auto launch = vec ? bn_bwd_launch<T, Vec16<T>::N> : bn_bwd_launch<T, 1>;
    return launch(dy, z, gamma, beta, mean, invstd, dz, dgamma_dbeta, R, (int)C, slope, training, workspace, st);
  });
}
