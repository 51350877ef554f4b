// The implicit-GEMM main loop shared by the image convolutions of libdva_conv2d.so (conv2d.cu) and libdva_unet.so
// (conv2d_up.cu).  Device code only: each library defines its own __global__ kernels, in its own namespace, and
// passes the main loop its operand gathers (the taps of a convolution, rows of a filter) as functors; the epilogue
// is the kernel's own code over the accumulator fragment (acc_row / acc_col name the element each register holds).
//
//   64 x 64 output tile, 4 warps of 32 x 32, k-tiles of 16 staged through registers into double-buffered shared
//   memory; mma.sync.m16n8k8 in 3xTF32 (a = hi + lo, a.b ~ lo.hi + hi.lo + hi.hi in fp32: fp32-grade).
#pragma once
#include <cstdint>

namespace dva_convgemm {

constexpr int kThreads = 128;
constexpr int BM = 64, BN = 64, BK = 16, LDS = BK + 4;   // LDS = 4 mod 8 words: conflict-free fragment loads
constexpr int kRedThreads = 256;

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

}  // namespace dva_convgemm
