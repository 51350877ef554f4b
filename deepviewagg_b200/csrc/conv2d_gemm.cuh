// The code shared by the image convolutions of libdva_conv2d.so (conv2d.cu), libdva_unet.so (conv2d_up.cu) and
// libdva_resnet.so (resnet.cu): the implicit-GEMM main loop, the device helpers of their epilogues and reductions,
// and the host-side sizing of their grids.  Each library defines its own __global__ kernels, in its own namespace,
// and passes the main loop its operand gathers (the taps of a convolution, rows of a filter) as functors; the
// epilogue is the kernel's own code over the accumulator fragment (acc_row / acc_col name the element each register
// holds), with column_stats / store_tile for the parts every library shares.
//
//   64 x 64 output tile, 4 warps of 32 x 32, k-tiles of 16 staged through registers into double-buffered shared
//   memory; mma.sync.m16n8k8 in 3xTF32 (a = hi + lo, a.b ~ lo.hi + hi.lo + hi.hi in fp32: fp32-grade).
#pragma once
#include "dva_common.cuh"
#include <algorithm>
#include <cstdint>

namespace dva_convgemm {

constexpr int kThreads = 128;
constexpr int BM = 64, BN = 64, BK = 16, LDS = BK + 4;   // LDS = 4 mod 8 words: conflict-free fragment loads
constexpr int kRedThreads = 256;
constexpr int kRows = 8;   // norm-backward reduction CTAs: 32 channels x kRows row lanes

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// fp64 sum of v over the CTA (kRedThreads threads) in a fixed tree order; the result is valid in thread 0
__device__ __forceinline__ double block_sum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kRedThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

// the tile row / column that acc[m][n][q] of gemm_mainloop holds in this thread
__device__ __forceinline__ int acc_row(int m, int q) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  return (warp >> 1) * 32 + m * 16 + (lane >> 2) + 8 * (q >> 1);
}
__device__ __forceinline__ int acc_col(int n, int q) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  return (warp & 1) * 32 + n * 8 + 2 * (lane & 3) + (q & 1);
}

// the pixel (oh[i], ow[i]) of each GEMM row (tid >> 4) + 8 i that the A gather of gemm_mainloop<false, *> asks this
// thread for, in a tile of rows from pixel p0 of a P-pixel image Wo wide; oh[i] = -1 past the image's last pixel
__device__ __forceinline__ void tile_pixels(int64_t p0, int64_t P, int64_t Wo, int (&oh)[8], int (&ow)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t p = p0 + ((int)threadIdx.x >> 4) + 8 * i;
    oh[i] = p < P ? (int)(p / Wo) : -1;
    ow[i] = p < P ? (int)(p - (p / Wo) * Wo) : 0;
  }
}

// forward epilogue: cs[n][j] / cq[n][j], this thread's sums of z and z^2 in column acc_col(n, j), summed over the
// warp's 32 rows (lanes of equal tq); colst[wm][col] then holds the sums of the tile's row half wm, for every thread
__device__ __forceinline__ void column_stats(double (&cs)[4][2], double (&cq)[4][2], double2 (&colst)[2][BN]) {
#pragma unroll
  for (int n = 0; n < 4; ++n)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        cs[n][j] += __shfl_xor_sync(0xffffffffu, cs[n][j], o);
        cq[n][j] += __shfl_xor_sync(0xffffffffu, cq[n][j], o);
      }
  if ((threadIdx.x & 31) < 4) {
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int j = 0; j < 2; ++j) colst[threadIdx.x >> 6][acc_col(n, j)] = make_double2(cs[n][j], cq[n][j]);
  }
  __syncthreads();
}

// wgrad epilogue: the split's fp32 partial tile, out[(i0 + row) * ld + j0 + col] for rows < `rows`, cols < `cols`
__device__ __forceinline__ void store_tile(const float (&acc)[2][4][4], int i0, int j0, int rows, int cols, int ld,
                                           float* out) {
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int o = i0 + acc_row(m, q), col = j0 + acc_col(n, q);
        if (o < rows && col < cols) out[(int64_t)o * ld + col] = acc[m][n][q];
      }
}

// the statistics tail: s and q, this thread's sums of x and x^2 over n values, summed over the CTA; thread 0 writes
// the mean and 1 / sqrt(var + eps).  Returns (mean, biased variance) in fp64, in every thread.
__device__ __forceinline__ double2 finish_stats(double s, double q, double n, float eps, float& mean, float& invstd,
                                                double* sh) {
  s = block_sum(s, sh);
  q = block_sum(q, sh);
  const double mu = s / n, var = fmax(q / n - mu * mu, 0.0);
  if (threadIdx.x == 0) {
    mean = (float)mu;
    invstd = (float)(1.0 / sqrt(var + (double)eps));
  }
  return make_double2(mu, var);
}

// weight standardisation of one filter f[0, n) (standardize_weights of image.py:39-50): (f - mean) / ((std + 1e-5) *
// sqrt(fan)), mean and unbiased std in fp64 over the filter, sqrt(fan) in fp32 as torch.Tensor([fan]) there.  One CTA
// of kRedThreads per filter; put(i, v) stores the standardised weight i wherever the kernel's layouts want it.
template <class Put>
__device__ __forceinline__ void standardize_filter(const float* f, int n, int fan, double* sh, Put put) {
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kRedThreads) s += (double)f[i];
  const double mu = block_sum(s, sh) / n;
  double q = 0.0;
  for (int i = threadIdx.x; i < n; i += kRedThreads) q += ((double)f[i] - mu) * ((double)f[i] - mu);
  const double sd = sqrt(block_sum(q, sh) / (n - 1));
  const double a = 1.0 / ((sd + 1e-5) * (double)sqrtf((float)fan));
  for (int i = threadIdx.x; i < n; i += kRedThreads) put(i, (float)(((double)f[i] - mu) * a));
}

// its backward: df[i] from grad(i), the gradient of the standardised weight i (fp64) wherever the kernel reads it
template <class Grad>
__device__ __forceinline__ void standardize_filter_bwd(const float* f, int n, int fan, double* sh, Grad grad,
                                                       float* df) {
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kRedThreads) s += (double)f[i];
  const double mu = block_sum(s, sh) / n;
  double q = 0.0, g1 = 0.0, g2 = 0.0;
  for (int i = threadIdx.x; i < n; i += kRedThreads) {
    const double d = (double)f[i] - mu, gi = grad(i);
    q += d * d;
    g1 += gi;
    g2 += gi * d;
  }
  q = block_sum(q, sh);
  g1 = block_sum(g1, sh);
  g2 = block_sum(g2, sh);
  const double sd = sqrt(q / (n - 1)), den = sd + 1e-5;
  const double a = 1.0 / (den * (double)sqrtf((float)fan));
  // a filter of equal weights (q = 0, so g2 = 0 and sd = 0) has no std term: torch's std backward masks std == 0
  const double k2 = q > 0.0 ? a / den * g2 / ((n - 1) * sd) : 0.0;
  for (int i = threadIdx.x; i < n; i += kRedThreads) {
    const double d = (double)f[i] - mu;
    df[i] = (float)(a * (grad(i) - g1 / n) - k2 * d);
  }
}

// norm-backward CTAs of 32 channel lanes tx x kRows row lanes ty: the (s1, s2) of channel lane tx's row lanes folded
// into row lane 0 in row order.  Returns true in row lane 0 of a live channel lane, where s1 and s2 hold the result.
__device__ __forceinline__ bool fold_rows(double2 (&sh)[kRows][32], int tx, int ty, bool live, double& s1,
                                          double& s2) {
  sh[ty][tx] = make_double2(s1, s2);
  __syncthreads();
  if (ty != 0 || !live) return false;
  for (int r = 1; r < kRows; ++r) {
    s1 += sh[r][tx].x;
    s2 += sh[r][tx].y;
  }
  return true;
}

// D[64 x 64] += A[64 x k] . B[64 x k]^T over k in [k_begin, k_end).  fa(i, row, k) / fb(i, row, k) return the
// thread's i-th element of a k-tile (0 outside the operand).  A_ROWFAST / B_ROWFAST: consecutive threads walk the
// tile's rows (the operand is contiguous along them) instead of its k.
template <bool A_ROWFAST, bool B_ROWFAST, class FA, class FB>
__device__ __forceinline__ void gemm_mainloop(FA fa, FB fb, int64_t k_begin, int64_t k_end, float* smem,
                                              float (&acc)[2][4][4]) {
  float* As = smem;                 // [2][BM][LDS]
  float* Bs = smem + 2 * BM * LDS;  // [2][BN][LDS]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1, g = lane >> 2, tq = lane & 3;
  float ra[8], rb[8];
  auto fetch = [&](int64_t k0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = tid + i * kThreads;
      const int row = A_ROWFAST ? (e & 63) : (e >> 4), kk = A_ROWFAST ? (e >> 6) : (e & 15);
      ra[i] = k0 + kk < k_end ? fa(i, row, k0 + kk) : 0.f;
      const int rowb = B_ROWFAST ? (e & 63) : (e >> 4), kb = B_ROWFAST ? (e >> 6) : (e & 15);
      rb[i] = k0 + kb < k_end ? fb(i, rowb, k0 + kb) : 0.f;
    }
  };
  auto put = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = tid + i * kThreads;
      const int row = A_ROWFAST ? (e & 63) : (e >> 4), kk = A_ROWFAST ? (e >> 6) : (e & 15);
      As[buf * BM * LDS + row * LDS + kk] = ra[i];
      const int rowb = B_ROWFAST ? (e & 63) : (e >> 4), kb = B_ROWFAST ? (e >> 6) : (e & 15);
      Bs[buf * BN * LDS + rowb * LDS + kb] = rb[i];
    }
  };
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[m][n][q] = 0.f;
  if (k_begin >= k_end) return;
  fetch(k_begin);
  put(0);
  __syncthreads();
  int buf = 0;
  for (int64_t k0 = k_begin; k0 < k_end; k0 += BK) {
    const bool more = k0 + BK < k_end;
    if (more) fetch(k0 + BK);
    const float* A = As + buf * BM * LDS;
    const float* Bt = Bs + buf * BN * LDS;
#pragma unroll
    for (int ks = 0; ks < BK; ks += 8) {
      uint32_t ahi[2][4], alo[2][4], bhi[4][2], blo[4][2];
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const float* a = A + (wm * 32 + m * 16 + g) * LDS + ks + tq;
        const float v[4] = {a[0], a[8 * LDS], a[4], a[8 * LDS + 4]};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          ahi[m][q] = to_tf32(v[q]);
          alo[m][q] = to_tf32(v[q] - __uint_as_float(ahi[m][q]));
        }
      }
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        const float* b = Bt + (wn * 32 + n * 8 + g) * LDS + ks + tq;
        const float v[2] = {b[0], b[4]};
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          bhi[n][q] = to_tf32(v[q]);
          blo[n][q] = to_tf32(v[q] - __uint_as_float(bhi[n][q]));
        }
      }
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          mma_tf32(acc[m][n], alo[m], bhi[n][0], bhi[n][1]);
          mma_tf32(acc[m][n], ahi[m], blo[n][0], blo[n][1]);
          mma_tf32(acc[m][n], ahi[m], bhi[n][0], bhi[n][1]);
        }
    }
    if (more) put(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }
}

// ---- host-side sizes
inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline int elementwise_grid(int64_t n) { return dva::grid_cap(n, kRedThreads, 8); }

// split-K of a weight gradient over M GEMM rows with tiles_mn output tiles: enough splits for about 4 CTAs per SM, at
// least 4 k-tiles each, rows rounded to whole k-tiles
struct SplitRows {
  int64_t rows_per_split;
  int splits;
};
inline SplitRows split_rows(int64_t M, int64_t tiles_mn) {
  const int64_t want = std::max<int64_t>(1, cdiv(4 * dva::kNumSMs, tiles_mn));
  const int64_t splits = std::min<int64_t>(want, cdiv(M, 4 * BK));
  SplitRows s;
  s.rows_per_split = cdiv(cdiv(M, splits), BK) * BK;
  s.splits = (int)cdiv(M, s.rows_per_split);
  return s;
}

}  // namespace dva_convgemm
