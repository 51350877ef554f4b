// The dilated ResNet-18 image encoder pretrained on ADE20K (libdva_resnet.so, C ABI include/dva_resnet.h):
// zero-padded, strided and dilated convolutions with train-mode BatchNorm statistics in their epilogue, BatchNorm
// apply / backward, the stem's max pool and the wrappers' bilinear resize.
//
//   rn_weight_prep_kernel  w [Co][Ci][T][T] -> the forward's K-major filter and the data gradient's.
//   rn_conv_gemm_kernel<MODE>  the main loop of conv2d_gemm.cuh (64 x 64 tiles, mma.sync in 3xTF32); the A operand
//        is gathered on the fly (implicit GEMM) over the flat pixel rows of all images:
//          kFwd    taps (r, s) of x at (oh * stride - pad + r * dil, ...), 0 in the padding
//          kDgrad  taps of dz reaching input pixel ih: (ih + pad - r * dil) / stride where it divides
//        The forward epilogue takes per-(tile, channel) fp64 sums of z and z^2 (training only).
//   rn_bn_stats_kernel  one CTA per channel: the tile partials in a fixed order -> mean, invstd, and the running
//        stats updated as F.batch_norm does; in eval mode mean / invstd from the running stats.
//   rn_conv_wgrad_kernel + rn_wgrad_reduce_kernel  dW = dz^T . im2col(x) split over the output pixels, one fp32
//        partial per split, summed in fp64 in split order into the torch layout.
//   rn_bn_apply_kernel  y = relu(BN(z) [+ skip] [+ BN_s(zs)]) in one pass.
//   rn_bn_bwd_partial_kernel -> rn_bn_bwd_reduce_kernel -> rn_bn_bwd_dz_kernel  per-channel sums of g and g * zhat
//        over pixel chunks (g = dy masked by the saved output), reduced in chunk order; dgamma, dbeta, dz.
//   rn_maxpool_kernel / rn_maxpool_bwd_kernel  3x3 / 2 / 1 with the window position of the max; the backward is a
//        gather over the <= 4 windows covering a pixel.
//   rn_resize_kernel / rn_resize_bwd_kernel  bilinear, align_corners=False, torch's source index; the forward writes a
//        column slice of a wider row, the backward gathers over the output pixels that read each input pixel.
// Nothing that is summed uses atomics: every result is bitwise reproducible run to run.
#include "dva_common.cuh"
#include "../../include/dva_resnet.h"
#include "conv2d_gemm.cuh"
#include <algorithm>
#include <cmath>

// namespace dva_resnet: the kernels of libdva_resnet.so (case table: tests/test_resnet18_matrix_table.py)
namespace dva_resnet {
using namespace dva;
using namespace dva_convgemm;

enum { kFwd = 0, kDgrad = 1 };

struct ConvArgs {
  const float* src;   // the gathered operand: x (forward) or dz (data gradient)
  const float* wt;    // [N][K]
  const float* add;   // data gradient: out = acc + add
  float* out;         // [M][N]
  double2* part;      // forward, training: [N][tiles] (sum, sum of squares)
  int64_t M;          // GEMM rows: B * Ho * Wo
  int H, W;           // spatial size of src
  int Ho, Wo;         // the grid of GEMM rows per image
  int Cs, N, K, T, stride, dil, pad, tiles;
};

template <int MODE>
__global__ void __launch_bounds__(kThreads) rn_conv_gemm_kernel(ConvArgs a) {
  __shared__ __align__(16) float smem[2 * (BM + BN) * LDS];
  __shared__ double2 colst[2][BN];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, g = lane >> 2;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int64_t P = (int64_t)a.Ho * a.Wo;
  int oh[8], ow[8];
  int64_t img[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + (tid >> 4) + 8 * i;
    const int64_t b = m / P, p = m - b * P;
    oh[i] = m < a.M ? (int)(p / a.Wo) : -1;
    ow[i] = (int)(p - (p / a.Wo) * a.Wo);
    img[i] = b * a.H * a.W;
  }
  const int H = a.H, W = a.W, Cs = a.Cs, T = a.T;
  auto fa = [&](int i, int, int64_t k64) -> float {
    if (oh[i] < 0) return 0.f;
    const int k = (int)k64;
    const int r = k / (T * Cs), rem = k - r * T * Cs, s = rem / Cs, c = rem - s * Cs;
    int ih, iw;
    if (MODE == kFwd) {
      ih = oh[i] * a.stride - a.pad + r * a.dil;
      iw = ow[i] * a.stride - a.pad + s * a.dil;
    } else {
      const int th = oh[i] + a.pad - r * a.dil, tw = ow[i] + a.pad - s * a.dil;
      if (th < 0 || tw < 0 || th % a.stride != 0 || tw % a.stride != 0) return 0.f;
      ih = th / a.stride;
      iw = tw / a.stride;
    }
    if (ih < 0 || ih >= H || iw < 0 || iw >= W) return 0.f;
    return __ldg(a.src + (img[i] + (int64_t)ih * W + iw) * Cs + c);
  };
  auto fb = [&](int, int row, int64_t k) -> float {
    const int n = n0 + row;
    return n < a.N ? __ldg(a.wt + (int64_t)n * a.K + k) : 0.f;
  };
  float acc[2][4][4];
  gemm_mainloop<false, false>(fa, fb, 0, a.K, smem, acc);

  double cs[4][2], cq[4][2];
#pragma unroll
  for (int n = 0; n < 4; ++n) cs[n][0] = cs[n][1] = cq[n][0] = cq[n][1] = 0.0;
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int64_t row = m0 + acc_row(m, q);
        const int col = n0 + acc_col(n, q);
        if (row >= a.M || col >= a.N) continue;
        float v = acc[m][n][q];
        const int64_t o = row * a.N + col;
        if (MODE == kDgrad && a.add) v += a.add[o];
        a.out[o] = v;
        if (MODE == kFwd) {
          cs[n][q & 1] += (double)v;
          cq[n][q & 1] += (double)v * (double)v;
        }
      }
  if (MODE == kFwd && a.part) {
    // column sums over the warp's 32 rows (lanes of equal tq), then over the two row halves
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          cs[n][j] += __shfl_xor_sync(0xffffffffu, cs[n][j], o);
          cq[n][j] += __shfl_xor_sync(0xffffffffu, cq[n][j], o);
        }
    if (g == 0) {
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int j = 0; j < 2; ++j) colst[wm][acc_col(n, j)] = make_double2(cs[n][j], cq[n][j]);
    }
    __syncthreads();
    if (tid < BN && n0 + tid < a.N)
      a.part[(int64_t)(n0 + tid) * a.tiles + blockIdx.x] =
          make_double2(colst[0][tid].x + colst[1][tid].x, colst[0][tid].y + colst[1][tid].y);
  }
}

// one CTA per channel: the tile partials in a fixed order (training) or the running stats (eval)
__global__ void __launch_bounds__(kRedThreads)
rn_bn_stats_kernel(const double2* __restrict__ part, int tiles, int64_t n, int training, float momentum, float eps,
                   float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ mean,
                   float* __restrict__ invstd) {
  __shared__ double sh[kRedThreads];
  const int c = blockIdx.x;
  if (!training) {
    if (threadIdx.x == 0) {
      mean[c] = running_mean[c];
      invstd[c] = (float)(1.0 / sqrt((double)running_var[c] + (double)eps));
    }
    return;
  }
  double s = 0.0, q = 0.0;
  for (int t = threadIdx.x; t < tiles; t += kRedThreads) {
    const double2 d = part[(int64_t)c * tiles + t];
    s += d.x;
    q += d.y;
  }
  s = block_sum(s, sh);
  q = block_sum(q, sh);
  if (threadIdx.x == 0) {
    const double nn = (double)n, mu = s / nn;
    const double var = fmax(q / nn - mu * mu, 0.0);
    mean[c] = (float)mu;
    invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
    const double mo = (double)momentum;
    running_mean[c] = (float)((1.0 - mo) * (double)running_mean[c] + mo * mu);
    running_var[c] = (float)((1.0 - mo) * (double)running_var[c] + mo * var * nn / (nn - 1.0));
  }
}

struct WgradArgs {
  const float* dz;    // [B * Ho * Wo, Co]
  const float* x;     // [B * H * W, Ci]
  float* part;        // [splits][Co][Kd]
  int64_t M, rows_per_split;
  int H, W, Ho, Wo, Ci, Co, Kd, T, stride, dil, pad;
};

// D[oc][j] = sum over the split's output pixels m of dz[m][oc] * im2col(x)[m][j], j = (r * T + s) * Ci + c
__global__ void __launch_bounds__(kThreads) rn_conv_wgrad_kernel(WgradArgs a) {
  __shared__ __align__(16) float smem[2 * (BM + BN) * LDS];
  const int i0 = blockIdx.x * BM, j0 = blockIdx.y * BN;
  const int64_t m_begin = (int64_t)blockIdx.z * a.rows_per_split;
  const int64_t m_end = min(a.M, m_begin + a.rows_per_split);
  const int oc = i0 + (threadIdx.x & 63), j = j0 + (threadIdx.x & 63);
  const int r = j / (a.T * a.Ci), rem = j - r * a.T * a.Ci, s = rem / a.Ci, c = rem - s * a.Ci;
  const int64_t P = (int64_t)a.Ho * a.Wo;
  auto fa = [&](int, int, int64_t m) -> float { return oc < a.Co ? __ldg(a.dz + m * a.Co + oc) : 0.f; };
  auto fb = [&](int, int, int64_t m) -> float {
    if (j >= a.Kd) return 0.f;
    const int64_t bb = m / P, p = m - bb * P;
    const int oh = (int)(p / a.Wo), ow = (int)(p - (p / a.Wo) * a.Wo);
    const int ih = oh * a.stride - a.pad + r * a.dil, iw = ow * a.stride - a.pad + s * a.dil;
    if (ih < 0 || ih >= a.H || iw < 0 || iw >= a.W) return 0.f;
    return __ldg(a.x + ((bb * a.H + ih) * a.W + iw) * a.Ci + c);
  };
  float acc[2][4][4];
  gemm_mainloop<true, true>(fa, fb, m_begin, m_end, smem, acc);
  float* out = a.part + (int64_t)blockIdx.z * a.Co * a.Kd;
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int o = i0 + acc_row(m, q), col = j0 + acc_col(n, q);
        if (o < a.Co && col < a.Kd) out[(int64_t)o * a.Kd + col] = acc[m][n][q];
      }
}

// dw [Co][Ci][T][T]: the split partials [splits][Co][(r * T + s) * Ci + c] summed in fp64, in split order
__global__ void __launch_bounds__(kRedThreads)
rn_wgrad_reduce_kernel(const float* __restrict__ part, int splits, int Co, int Ci, int T, float* __restrict__ dw) {
  const int TT = T * T, Kd = TT * Ci;
  const int64_t n = (int64_t)Co * Kd;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = e / Kd;
    const int rem = (int)(e - o * Kd), c = rem / TT, rs = rem - c * TT;
    const int64_t src = o * Kd + (int64_t)rs * Ci + c;
    double s = 0.0;
    for (int z = 0; z < splits; ++z) s += (double)part[(int64_t)z * n + src];
    dw[e] = (float)s;
  }
}

// w [Co][Ci][T][T] -> wf [Co][T][T][Ci], wd [Ci][T][T][Co]
__global__ void __launch_bounds__(kRedThreads)
rn_weight_prep_kernel(const float* __restrict__ w, int Co, int Ci, int T, float* __restrict__ wf,
                      float* __restrict__ wd) {
  const int TT = T * T;
  const int64_t n = (int64_t)Co * Ci * TT;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = e / (Ci * TT);
    const int rem = (int)(e - o * Ci * TT), c = rem / TT, rs = rem - c * TT;
    const float v = w[e];
    wf[(o * TT + rs) * Ci + c] = v;
    wd[((int64_t)c * TT + rs) * Co + o] = v;
  }
}

__global__ void __launch_bounds__(kRedThreads)
rn_bn_apply_kernel(const float* __restrict__ z, int C, const float* __restrict__ mean,
                   const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                   const float* __restrict__ skip, const float* __restrict__ zs, const float* __restrict__ mean_s,
                   const float* __restrict__ invstd_s, const float* __restrict__ gamma_s,
                   const float* __restrict__ beta_s, float* __restrict__ y, int64_t n) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    float v = (z[e] - mean[c]) * invstd[c] * gamma[c] + beta[c];
    if (skip) v += skip[e];
    if (zs) v += (zs[e] - mean_s[c]) * invstd_s[c] * gamma_s[c] + beta_s[c];
    y[e] = fmaxf(v, 0.f);
  }
}

constexpr int kBnRows = 8;   // BatchNorm backward CTAs: 32 channels x 8 row lanes

__device__ __forceinline__ float masked(float dy, float y) { return y > 0.f ? dy : 0.f; }

// per (chunk of pixels, channel): sums of g and g * zhat
__global__ void __launch_bounds__(32 * kBnRows)
rn_bn_bwd_partial_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ z,
                         int64_t M, int C, const float* __restrict__ mean, const float* __restrict__ invstd,
                         int64_t rows_per_chunk, double2* __restrict__ part) {
  __shared__ double2 sh[kBnRows][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.y * 32 + tx;
  const int64_t chunk = blockIdx.x;
  double s1 = 0.0, s2 = 0.0;
  if (c < C) {
    const float mu = mean[c], is = invstd[c];
    const int64_t m_end = min(M, (chunk + 1) * rows_per_chunk);
    for (int64_t m = chunk * rows_per_chunk + ty; m < m_end; m += kBnRows) {
      const int64_t e = m * C + c;
      const float gv = masked(dy[e], y[e]);
      s1 += (double)gv;
      s2 += (double)gv * (double)((z[e] - mu) * is);
    }
  }
  sh[ty][tx] = make_double2(s1, s2);
  __syncthreads();
  if (ty == 0 && c < C) {
    for (int r = 1; r < kBnRows; ++r) {
      s1 += sh[r][tx].x;
      s2 += sh[r][tx].y;
    }
    part[chunk * C + c] = make_double2(s1, s2);
  }
}

// per channel: the chunk partials in chunk order -> dbeta, dgamma and the means of g and g * zhat (training)
__global__ void __launch_bounds__(32 * kBnRows)
rn_bn_bwd_reduce_kernel(const double2* __restrict__ part, int64_t chunks, int C, int64_t M, int training,
                        float* __restrict__ dgamma, float* __restrict__ dbeta, double2* __restrict__ coef) {
  __shared__ double2 sh[kBnRows][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  double s1 = 0.0, s2 = 0.0;
  if (c < C)
    for (int64_t k = ty; k < chunks; k += kBnRows) {
      const double2 d = part[k * C + c];
      s1 += d.x;
      s2 += d.y;
    }
  sh[ty][tx] = make_double2(s1, s2);
  __syncthreads();
  if (ty == 0 && c < C) {
    for (int r = 1; r < kBnRows; ++r) {
      s1 += sh[r][tx].x;
      s2 += sh[r][tx].y;
    }
    dbeta[c] = (float)s1;
    dgamma[c] = (float)s2;
    coef[c] = training ? make_double2(s1 / (double)M, s2 / (double)M) : make_double2(0.0, 0.0);
  }
}

__global__ void __launch_bounds__(kRedThreads)
rn_bn_bwd_dz_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ z, int C,
                    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                    const double2* __restrict__ coef, float* __restrict__ dz, float* __restrict__ gout, int64_t n) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    const float gv = masked(dy[e], y[e]);
    const float is = invstd[c];
    const double2 k = coef[c];
    const double zh = (double)((z[e] - mean[c]) * is);
    dz[e] = (float)((double)gamma[c] * (double)is * ((double)gv - k.x - zh * k.y));
    if (gout) gout[e] = gv;
  }
}

// one thread per output element; the window's first valid tap starts as the max (as torch's max_pool2d)
__global__ void __launch_bounds__(kRedThreads)
rn_maxpool_kernel(const float* __restrict__ x, int H, int W, int Ho, int Wo, int C, float* __restrict__ y,
                  uint8_t* __restrict__ arg, int64_t n) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pix = e / C;
    const int c = (int)(e - pix * C);
    const int64_t b = pix / ((int64_t)Ho * Wo);
    const int p = (int)(pix - b * Ho * Wo), oh = p / Wo, ow = p - oh * Wo;
    const int h0 = 2 * oh - 1, w0 = 2 * ow - 1;
    const float* xb = x + b * H * W * (int64_t)C + c;
    float mx = -INFINITY;
    int best = (h0 < 0 ? 3 : 0) + (w0 < 0 ? 1 : 0);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ih = h0 + r, iw = w0 + s;
        if (ih < 0 || ih >= H || iw < 0 || iw >= W) continue;
        const float v = __ldg(xb + ((int64_t)ih * W + iw) * C);
        if (v > mx || isnan(v)) {
          mx = v;
          best = r * 3 + s;
        }
      }
    y[e] = mx;
    arg[e] = (uint8_t)best;
  }
}

// one thread per input element: the windows (oh, ow) covering (ih, iw) in row-major order
__global__ void __launch_bounds__(kRedThreads)
rn_maxpool_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ arg, int H, int W, int Ho, int Wo,
                      int C, float* __restrict__ dx, int64_t n) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pix = e / C;
    const int c = (int)(e - pix * C);
    const int64_t b = pix / ((int64_t)H * W);
    const int p = (int)(pix - b * H * W), ih = p / W, iw = p - ih * W;
    float v = 0.f;
#pragma unroll
    for (int r = 2; r >= 0; --r) {
      const int th = ih + 1 - r;
      if (th < 0 || (th & 1) || th / 2 >= Ho) continue;
#pragma unroll
      for (int s = 2; s >= 0; --s) {
        const int tw = iw + 1 - s;
        if (tw < 0 || (tw & 1) || tw / 2 >= Wo) continue;
        const int64_t o = ((b * Ho + th / 2) * Wo + tw / 2) * C + c;
        if (arg[o] == r * 3 + s) v += dy[o];
      }
    }
    dx[e] = v;
  }
}

// torch's bilinear source index (align_corners=False): lower tap, upper tap, and their weights
struct Taps {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Taps taps(float scale, int o, int in) {
  float src = scale * ((float)o + 0.5f) - 0.5f;
  src = src < 0.f ? 0.f : src;
  Taps t;
  t.i0 = (int)src;
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  t.l1 = src - (float)t.i0;
  t.l0 = 1.f - t.l1;
  return t;
}
__device__ __forceinline__ float weight_of(const Taps& t, int i) {
  return (t.i0 == i ? t.l0 : 0.f) + (t.i1 == i ? t.l1 : 0.f);
}
// the output indices reading input i: [first o with i1(o) >= i, last o with i0(o) <= i] (both are monotone)
__device__ __forceinline__ int2 readers(float scale, int i, int in, int out) {
  int lo = 0, hi = out;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (taps(scale, mid, in).i1 >= i) hi = mid; else lo = mid + 1;
  }
  int lo2 = lo, hi2 = out;
  while (lo2 < hi2) {
    const int mid = (lo2 + hi2) >> 1;
    if (taps(scale, mid, in).i0 > i) hi2 = mid; else lo2 = mid + 1;
  }
  return make_int2(lo, lo2);
}

__global__ void __launch_bounds__(kRedThreads)
rn_resize_kernel(const float* __restrict__ x, int H, int W, int C, int Ho, int Wo, float sh, float sw,
                 float* __restrict__ y, int64_t ldy, int64_t col0, int64_t n) {
  const bool same = H == Ho && W == Wo;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pix = e / C;
    const int c = (int)(e - pix * C);
    const int64_t b = pix / ((int64_t)Ho * Wo);
    const int p = (int)(pix - b * Ho * Wo), oh = p / Wo, ow = p - oh * Wo;
    const float* xb = x + b * H * W * (int64_t)C + c;
    float v;
    if (same) {
      v = __ldg(xb + (int64_t)p * C);
    } else {
      const Taps th = taps(sh, oh, H), tw = taps(sw, ow, W);
      const float a = tw.l0 * __ldg(xb + ((int64_t)th.i0 * W + tw.i0) * C) +
                      tw.l1 * __ldg(xb + ((int64_t)th.i0 * W + tw.i1) * C);
      const float d = tw.l0 * __ldg(xb + ((int64_t)th.i1 * W + tw.i0) * C) +
                      tw.l1 * __ldg(xb + ((int64_t)th.i1 * W + tw.i1) * C);
      v = th.l0 * a + th.l1 * d;
    }
    y[pix * ldy + col0 + c] = v;
  }
}

__global__ void __launch_bounds__(kRedThreads)
rn_resize_bwd_kernel(const float* __restrict__ dy, int64_t ldy, int64_t col0, int H, int W, int C, int Ho, int Wo,
                     float sh, float sw, float* __restrict__ dx, int64_t n) {
  const bool same = H == Ho && W == Wo;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pix = e / C;
    const int c = (int)(e - pix * C);
    const int64_t b = pix / ((int64_t)H * W);
    const int p = (int)(pix - b * H * W), ih = p / W, iw = p - ih * W;
    const float* gb = dy + b * Ho * (int64_t)Wo * ldy + col0 + c;
    float v = 0.f;
    if (same) {
      v = gb[(int64_t)p * ldy];
    } else {
      const int2 rh = readers(sh, ih, H, Ho), rw = readers(sw, iw, W, Wo);
      for (int oh = rh.x; oh < rh.y; ++oh) {
        const float wh = weight_of(taps(sh, oh, H), ih);
        float row = 0.f;
        for (int ow = rw.x; ow < rw.y; ++ow)
          row += weight_of(taps(sw, ow, W), iw) * gb[((int64_t)oh * Wo + ow) * ldy];
        v += wh * row;
      }
    }
    dx[e] = v;
  }
}

// ---- host-side sizes
inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline int64_t out_size(int64_t n, int stride) { return (n - 1) / stride + 1; }
inline int pad_of(int T, int dil) { return T == 3 ? dil : 0; }

inline int check_conv(const char* what, int64_t B, int64_t H, int64_t W, int Ci, int Co, int T, int stride, int dil) {
  const bool ok = (T == 3 && stride == 1 && (dil == 1 || dil == 2 || dil == 4)) ||
                  (T == 3 && stride == 2 && dil == 1) || (T == 1 && (stride == 1 || stride == 2) && dil == 1);
  if (!ok) return failf(DVA_EINVAL, "%s: unsupported shape (T %d, stride %d, dilation %d)", what, T, stride, dil);
  if (B < 1 || H < 1 || W < 1 || Ci < 1 || Co < 1) return failf(DVA_EINVAL, "%s: bad sizes", what);
  if ((int64_t)Co * T * T * Ci > (int64_t)INT32_MAX / 4 || H > INT32_MAX / 8 || W > INT32_MAX / 8)
    return failf(DVA_EUNSUPPORTED, "%s: sizes beyond the 32-bit index range", what);
  if (cdiv(B * H * W, BM) > INT32_MAX) return failf(DVA_EUNSUPPORTED, "%s: too many pixels", what);
  return DVA_OK;
}

struct WgradPlan {
  int64_t M, rows_per_split;
  int splits, Kd;
};
inline WgradPlan wgrad_plan(int64_t B, int64_t H, int64_t W, int Ci, int Co, int T, int stride) {
  WgradPlan p;
  p.M = B * out_size(H, stride) * out_size(W, stride);
  p.Kd = T * T * Ci;
  const int64_t tiles_mn = cdiv(Co, BM) * cdiv(p.Kd, BN);
  const int64_t want = std::max<int64_t>(1, cdiv(4 * kNumSMs, tiles_mn));
  const int64_t splits = std::min<int64_t>(want, cdiv(p.M, 4 * BK));
  p.rows_per_split = cdiv(cdiv(p.M, splits), BK) * BK;
  p.splits = (int)cdiv(p.M, p.rows_per_split);
  return p;
}

struct BnPlan {
  int64_t chunks, rows_per_chunk;
};
inline BnPlan bn_plan(int64_t M, int C) {
  BnPlan p;
  const int64_t cap = std::max<int64_t>(1, 2048 / cdiv(C, 32));
  p.chunks = std::max<int64_t>(1, std::min<int64_t>(cdiv(M, 256), cap));
  p.rows_per_chunk = cdiv(M, p.chunks);
  p.chunks = cdiv(M, p.rows_per_chunk);
  return p;
}

inline int elementwise_grid(int64_t n) { return grid_cap(n, kRedThreads, 8); }

}  // namespace dva_resnet

using namespace dva;
using namespace dva_resnet;

extern "C" int dva_resnet_weight_prep(const float* w, int Co, int Ci, int T, float* wf, float* wd, void* stream) {
  if (T != 1 && T != 3) return fail(DVA_EINVAL, "resnet_weight_prep: T must be 1 or 3");
  if (Co < 1 || Ci < 1) return fail(DVA_EINVAL, "resnet_weight_prep: bad sizes");
  if (!w || !wf || !wd) return fail(DVA_EINVAL, "resnet_weight_prep: null pointer");
  const int64_t n = (int64_t)Co * Ci * T * T;
  rn_weight_prep_kernel<<<elementwise_grid(n), kRedThreads, 0, (cudaStream_t)stream>>>(w, Co, Ci, T, wf, wd);
  return check_launch("resnet_weight_prep");
}

extern "C" size_t dva_resnet_fwd_workspace_bytes(int64_t B, int64_t Ho, int64_t Wo, int Co) {
  if (B < 1 || Ho < 1 || Wo < 1 || Co < 1) return 0;
  return (size_t)cdiv(B * Ho * Wo, BM) * Co * sizeof(double2);
}

extern "C" int dva_resnet_conv_bn_fwd(const float* x, int64_t B, int64_t H, int64_t W, int Ci, const float* wf,
                                      int Co, int T, int stride, int dil, int training, float momentum, float eps,
                                      float* running_mean, float* running_var, float* z, float* mean, float* invstd,
                                      void* ws, size_t ws_bytes, void* stream) {
  const int rc = check_conv("resnet_conv_bn_fwd", B, H, W, Ci, Co, T, stride, dil);
  if (rc != DVA_OK) return rc;
  if (!x || !wf || !running_mean || !running_var || !z || !mean || !invstd)
    return fail(DVA_EINVAL, "resnet_conv_bn_fwd: null pointer");
  const int64_t Ho = out_size(H, stride), Wo = out_size(W, stride), M = B * Ho * Wo;
  if (training && M < 2) return fail(DVA_EINVAL, "resnet_conv_bn_fwd: training needs more than 1 value per channel");
  if (training && (!ws || ws_bytes < dva_resnet_fwd_workspace_bytes(B, Ho, Wo, Co)))
    return fail(DVA_EINVAL, "resnet_conv_bn_fwd: workspace too small");
  ConvArgs a{};
  a.src = x; a.wt = wf; a.out = z; a.part = training ? (double2*)ws : nullptr;
  a.M = M; a.H = (int)H; a.W = (int)W; a.Ho = (int)Ho; a.Wo = (int)Wo;
  a.Cs = Ci; a.N = Co; a.K = T * T * Ci; a.T = T; a.stride = stride; a.dil = dil; a.pad = pad_of(T, dil);
  a.tiles = (int)cdiv(M, BM);
  cudaStream_t st = (cudaStream_t)stream;
  rn_conv_gemm_kernel<kFwd><<<dim3((unsigned)a.tiles, (unsigned)cdiv(Co, BN)), kThreads, 0, st>>>(a);
  const int r2 = check_launch("resnet_conv_bn_fwd");
  if (r2 != DVA_OK) return r2;
  rn_bn_stats_kernel<<<Co, kRedThreads, 0, st>>>(a.part, a.tiles, M, training, momentum, eps, running_mean,
                                                 running_var, mean, invstd);
  return check_launch("resnet_conv_bn_fwd_stats");
}

extern "C" int dva_resnet_conv_dgrad(const float* dz, int64_t B, int64_t H, int64_t W, int Ci, int Co,
                                     const float* wd, int T, int stride, int dil, const float* add, float* dx,
                                     void* stream) {
  const int rc = check_conv("resnet_conv_dgrad", B, H, W, Ci, Co, T, stride, dil);
  if (rc != DVA_OK) return rc;
  if (!dz || !wd || !dx) return fail(DVA_EINVAL, "resnet_conv_dgrad: null pointer");
  ConvArgs a{};
  a.src = dz; a.wt = wd; a.add = add; a.out = dx;
  a.M = B * H * W; a.H = (int)out_size(H, stride); a.W = (int)out_size(W, stride); a.Ho = (int)H; a.Wo = (int)W;
  a.Cs = Co; a.N = Ci; a.K = T * T * Co; a.T = T; a.stride = stride; a.dil = dil; a.pad = pad_of(T, dil);
  a.tiles = (int)cdiv(a.M, BM);
  rn_conv_gemm_kernel<kDgrad><<<dim3((unsigned)a.tiles, (unsigned)cdiv(Ci, BN)), kThreads, 0, (cudaStream_t)stream>>>(a);
  return check_launch("resnet_conv_dgrad");
}

extern "C" size_t dva_resnet_wgrad_workspace_bytes(int64_t B, int64_t H, int64_t W, int Ci, int Co, int T, int stride,
                                                   int dil) {
  if (B < 1 || H < 1 || W < 1 || Ci < 1 || Co < 1 || (T != 1 && T != 3) || stride < 1 || dil < 1) return 0;
  const WgradPlan p = wgrad_plan(B, H, W, Ci, Co, T, stride);
  return (size_t)p.splits * Co * p.Kd * sizeof(float);
}

extern "C" int dva_resnet_conv_wgrad(const float* dz, const float* x, int64_t B, int64_t H, int64_t W, int Ci, int Co,
                                     int T, int stride, int dil, float* dw, void* ws, size_t ws_bytes, void* stream) {
  const int rc = check_conv("resnet_conv_wgrad", B, H, W, Ci, Co, T, stride, dil);
  if (rc != DVA_OK) return rc;
  if (!dz || !x || !dw || !ws) return fail(DVA_EINVAL, "resnet_conv_wgrad: null pointer");
  if (ws_bytes < dva_resnet_wgrad_workspace_bytes(B, H, W, Ci, Co, T, stride, dil))
    return fail(DVA_EINVAL, "resnet_conv_wgrad: workspace too small");
  const WgradPlan pl = wgrad_plan(B, H, W, Ci, Co, T, stride);
  WgradArgs a{};
  a.dz = dz; a.x = x; a.part = (float*)ws; a.M = pl.M; a.rows_per_split = pl.rows_per_split;
  a.H = (int)H; a.W = (int)W; a.Ho = (int)out_size(H, stride); a.Wo = (int)out_size(W, stride);
  a.Ci = Ci; a.Co = Co; a.Kd = pl.Kd; a.T = T; a.stride = stride; a.dil = dil; a.pad = pad_of(T, dil);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)cdiv(Co, BM), (unsigned)cdiv(pl.Kd, BN), (unsigned)pl.splits);
  rn_conv_wgrad_kernel<<<grid, kThreads, 0, st>>>(a);
  const int r2 = check_launch("resnet_conv_wgrad");
  if (r2 != DVA_OK) return r2;
  rn_wgrad_reduce_kernel<<<elementwise_grid((int64_t)Co * pl.Kd), kRedThreads, 0, st>>>(a.part, pl.splits, Co, Ci, T,
                                                                                        dw);
  return check_launch("resnet_conv_wgrad_reduce");
}

extern "C" int dva_resnet_bn_apply(const float* z, int64_t M, int C, const float* mean, const float* invstd,
                                   const float* gamma, const float* beta, const float* skip, const float* zs,
                                   const float* mean_s, const float* invstd_s, const float* gamma_s,
                                   const float* beta_s, float* y, void* stream) {
  if (M < 1 || C < 1) return fail(DVA_EINVAL, "resnet_bn_apply: bad sizes");
  if (!z || !mean || !invstd || !gamma || !beta || !y) return fail(DVA_EINVAL, "resnet_bn_apply: null pointer");
  if (zs && (!mean_s || !invstd_s || !gamma_s || !beta_s)) return fail(DVA_EINVAL, "resnet_bn_apply: null pointer");
  const int64_t n = M * C;
  rn_bn_apply_kernel<<<elementwise_grid(n), kRedThreads, 0, (cudaStream_t)stream>>>(
      z, C, mean, invstd, gamma, beta, skip, zs, mean_s, invstd_s, gamma_s, beta_s, y, n);
  return check_launch("resnet_bn_apply");
}

extern "C" size_t dva_resnet_bn_bwd_workspace_bytes(int64_t M, int C) {
  if (M < 1 || C < 1) return 0;
  const BnPlan p = bn_plan(M, C);
  return round256((size_t)p.chunks * C * sizeof(double2)) + (size_t)C * sizeof(double2);
}

extern "C" int dva_resnet_bn_bwd(const float* dy, const float* y, const float* z, int64_t M, int C, const float* mean,
                                 const float* invstd, const float* gamma, int training, float* dz, float* gout,
                                 float* dgamma, float* dbeta, void* ws, size_t ws_bytes, void* stream) {
  if (M < 1 || C < 1) return fail(DVA_EINVAL, "resnet_bn_bwd: bad sizes");
  if (!dy || !y || !z || !mean || !invstd || !gamma || !dz || !dgamma || !dbeta || !ws)
    return fail(DVA_EINVAL, "resnet_bn_bwd: null pointer");
  if (ws_bytes < dva_resnet_bn_bwd_workspace_bytes(M, C)) return fail(DVA_EINVAL, "resnet_bn_bwd: workspace too small");
  const BnPlan pl = bn_plan(M, C);
  double2* part = (double2*)ws;
  double2* coef = (double2*)((uint8_t*)ws + round256((size_t)pl.chunks * C * sizeof(double2)));
  cudaStream_t st = (cudaStream_t)stream;
  const int cb = (int)cdiv(C, 32);
  rn_bn_bwd_partial_kernel<<<dim3((unsigned)pl.chunks, cb), 32 * kBnRows, 0, st>>>(dy, y, z, M, C, mean, invstd,
                                                                                   pl.rows_per_chunk, part);
  int rc = check_launch("resnet_bn_bwd_partial");
  if (rc != DVA_OK) return rc;
  rn_bn_bwd_reduce_kernel<<<cb, 32 * kBnRows, 0, st>>>(part, pl.chunks, C, M, training, dgamma, dbeta, coef);
  rc = check_launch("resnet_bn_bwd_reduce");
  if (rc != DVA_OK) return rc;
  const int64_t n = M * C;
  rn_bn_bwd_dz_kernel<<<elementwise_grid(n), kRedThreads, 0, st>>>(dy, y, z, C, mean, invstd, gamma, coef, dz, gout,
                                                                   n);
  return check_launch("resnet_bn_bwd_dz");
}

extern "C" int dva_resnet_maxpool(const float* x, int64_t B, int64_t H, int64_t W, int C, float* y, uint8_t* arg,
                                  void* stream) {
  if (B < 1 || H < 1 || W < 1 || C < 1) return fail(DVA_EINVAL, "resnet_maxpool: bad sizes");
  if (H > INT32_MAX / 4 || W > INT32_MAX / 4 || H * W > INT32_MAX)
    return fail(DVA_EUNSUPPORTED, "resnet_maxpool: sizes beyond the 32-bit index range");
  if (!x || !y || !arg) return fail(DVA_EINVAL, "resnet_maxpool: null pointer");
  const int64_t Ho = out_size(H, 2), Wo = out_size(W, 2), n = B * Ho * Wo * C;
  rn_maxpool_kernel<<<elementwise_grid(n), kRedThreads, 0, (cudaStream_t)stream>>>(x, (int)H, (int)W, (int)Ho,
                                                                                   (int)Wo, C, y, arg, n);
  return check_launch("resnet_maxpool");
}

extern "C" int dva_resnet_maxpool_bwd(const float* dy, const uint8_t* arg, int64_t B, int64_t H, int64_t W, int C,
                                      float* dx, void* stream) {
  if (B < 1 || H < 1 || W < 1 || C < 1) return fail(DVA_EINVAL, "resnet_maxpool_bwd: bad sizes");
  if (H > INT32_MAX / 4 || W > INT32_MAX / 4 || H * W > INT32_MAX)
    return fail(DVA_EUNSUPPORTED, "resnet_maxpool_bwd: sizes beyond the 32-bit index range");
  if (!dy || !arg || !dx) return fail(DVA_EINVAL, "resnet_maxpool_bwd: null pointer");
  const int64_t n = B * H * W * C;
  rn_maxpool_bwd_kernel<<<elementwise_grid(n), kRedThreads, 0, (cudaStream_t)stream>>>(
      dy, arg, (int)H, (int)W, (int)out_size(H, 2), (int)out_size(W, 2), C, dx, n);
  return check_launch("resnet_maxpool_bwd");
}

static int check_resize(const char* what, int64_t B, int64_t H, int64_t W, int C, int64_t Ho, int64_t Wo,
                        float scale_h, float scale_w, int64_t ldy, int64_t col0) {
  if (B < 1 || H < 1 || W < 1 || C < 1 || Ho < 1 || Wo < 1) return failf(DVA_EINVAL, "%s: bad sizes", what);
  if (!(scale_h > 0.f) || !(scale_w > 0.f) || !std::isfinite(scale_h) || !std::isfinite(scale_w))
    return failf(DVA_EINVAL, "%s: bad scale", what);
  if (col0 < 0 || col0 + C > ldy) return failf(DVA_EINVAL, "%s: the column slice does not fit the rows", what);
  if (H * W > INT32_MAX || Ho * Wo > INT32_MAX)
    return failf(DVA_EUNSUPPORTED, "%s: sizes beyond the 32-bit index range", what);
  return DVA_OK;
}

extern "C" int dva_resnet_resize(const float* x, int64_t B, int64_t H, int64_t W, int C, int64_t Ho, int64_t Wo,
                                 float scale_h, float scale_w, float* y, int64_t ldy, int64_t col0, void* stream) {
  const int rc = check_resize("resnet_resize", B, H, W, C, Ho, Wo, scale_h, scale_w, ldy, col0);
  if (rc != DVA_OK) return rc;
  if (!x || !y) return fail(DVA_EINVAL, "resnet_resize: null pointer");
  const int64_t n = B * Ho * Wo * C;
  rn_resize_kernel<<<elementwise_grid(n), kRedThreads, 0, (cudaStream_t)stream>>>(
      x, (int)H, (int)W, C, (int)Ho, (int)Wo, scale_h, scale_w, y, ldy, col0, n);
  return check_launch("resnet_resize");
}

extern "C" int dva_resnet_resize_bwd(const float* dy, int64_t ldy, int64_t col0, int64_t B, int64_t H, int64_t W,
                                     int C, int64_t Ho, int64_t Wo, float scale_h, float scale_w, float* dx,
                                     void* stream) {
  const int rc = check_resize("resnet_resize_bwd", B, H, W, C, Ho, Wo, scale_h, scale_w, ldy, col0);
  if (rc != DVA_OK) return rc;
  if (!dy || !dx) return fail(DVA_EINVAL, "resnet_resize_bwd: null pointer");
  const int64_t n = B * H * W * C;
  rn_resize_bwd_kernel<<<elementwise_grid(n), kRedThreads, 0, (cudaStream_t)stream>>>(
      dy, ldy, col0, (int)H, (int)W, C, (int)Ho, (int)Wo, scale_h, scale_w, dx, n);
  return check_launch("resnet_resize_bwd");
}
