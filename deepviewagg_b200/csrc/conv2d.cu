// The from-scratch image encoder (libdva_conv2d.so, C ABI include/dva_conv2d.h): weight-standardised implicit-GEMM
// convolutions with the GroupNorm statistics in their epilogue, and the GroupNorm / ReLUWS / residual pass.
//
//   weight_prep_kernel / weight_prep_bwd_kernel  one CTA per filter: mean and unbiased std over Ci*R*S in fp64
//        (image.py:39-50; sqrt(fan_in) in fp32, as torch.Tensor([C_in]) there), the standardised filter written in the forward's K-major layout and in the layout
//        the data gradient reads; the backward maps the gradient of that filter back to the torch layout.
//   conv_gemm_kernel<MODE>  the main loop of conv2d_gemm.cuh (64 x 64 tiles, mma.sync in 3xTF32: fp32-grade, as
//        skinny_gemm.cu).  The A operand is gathered on the fly (implicit GEMM):
//          kFwd3   3x3 reflect-padded taps of x            kFwd2   2x2 stride-2 taps of x       kFwd1  rows of x
//          kDgrad3 taps of dz, the reflected border folded back onto rows / columns 1 and H-2 / W-2
//          kDgrad2 rows of dz against [R][S][Ci] x Co, scattered to the one input pixel each tap reaches
//          kDgrad1 rows of dz
//        A tile never straddles two images, so the forward epilogue (bias, z, per-column fp64 sums of z and z^2
//        reduced to one partial per (tile, group)) needs no second pass over z.
//   gn_stats_kernel  one CTA per (image, group): the partials in a fixed order -> mean, invstd.
//   conv_wgrad_kernel<KIND> + wgrad_reduce_kernel  dW = dz^T . im2col(x) split over the output pixels, one fp32
//        partial per split, summed in fp64 in split order; a column of ones appended to im2col gives dbias.
//   gn_apply_kernel  y = act(GN(z)) [+ skip] [+ GN_s(zs)] in one pass.
//   gn_bwd_partial_kernel -> gn_bwd_sums_kernel -> gn_bwd_coef_kernel -> gn_bwd_dz_kernel  per (image, channel)
//        sums of g and g * zhat over pixel chunks, reduced in a fixed order; dgamma, dbeta and the per-(image,
//        group) coefficients of dz.
// Nothing that is summed uses atomics: every result is bitwise reproducible run to run.
#include "dva_common.cuh"
#include "../../include/dva_conv2d.h"
#include "conv2d_gemm.cuh"
#include <algorithm>

// namespace dva_conv2d: the kernels of libdva_conv2d.so (case table: tests/test_conv2d_matrix_table.py)
namespace dva_conv2d {
using namespace dva;
using namespace dva_convgemm;

enum { kFwd3 = 0, kFwd2 = 1, kFwd1 = 2, kDgrad3 = 3, kDgrad2 = 4, kDgrad1 = 5 };

__host__ __device__ __forceinline__ int taps_of(int kind) {
  return kind == DVA_CONV_3X3_REFLECT ? 3 : (kind == DVA_CONV_2X2_S2 ? 2 : 1);
}

__device__ __forceinline__ int reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

struct GemmArgs {
  const float* src;   // the gathered operand: x (forward) or dz (data gradient)
  const float* wt;    // [N][K]
  const float* bias;  // forward
  const float* add;   // data gradient: out = acc + add
  float* out;
  double2* part;      // forward: one (sum, sum of squares) per (tile, column tile, group)
  int64_t H, W;       // spatial size of src
  int64_t Ho, Wo;     // the grid of GEMM rows, per image (P = Ho * Wo)
  int64_t Hx, Wx;     // kDgrad2: spatial size of dx
  int Cs;             // channels of src
  int N, K;
  int G, cpg, tiles, ntiles;
};

template <int MODE>
__global__ void __launch_bounds__(kThreads) conv_gemm_kernel(GemmArgs a) {
  __shared__ __align__(16) float smem[2 * (BM + BN) * LDS];
  __shared__ double2 colst[2][BN];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1, g = lane >> 2, tq = lane & 3;
  const int64_t b = blockIdx.x / a.tiles;
  const int t = (int)(blockIdx.x - b * a.tiles);
  const int64_t P = a.Ho * a.Wo, p0 = (int64_t)t * BM;
  const int n0 = blockIdx.y * BN;
  const int64_t img = b * a.H * a.W;   // first source pixel of image b (gathering modes)
  const int64_t row0 = b * P + p0;     // first GEMM row of the tile
  int oh[8], ow[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t p = p0 + (tid >> 4) + 8 * i;
    oh[i] = p < P ? (int)(p / a.Wo) : -1;
    ow[i] = p < P ? (int)(p - (p / a.Wo) * a.Wo) : 0;
  }
  const int H = (int)a.H, W = (int)a.W, Cs = a.Cs, K = a.K;
  auto fa = [&](int i, int row, int64_t k64) -> float {
    if (oh[i] < 0) return 0.f;
    const int k = (int)k64;
    if (MODE == kFwd3 || MODE == kFwd2 || MODE == kDgrad3) {
      const int T = MODE == kFwd2 ? 2 : 3;
      const int r = k / (T * Cs), rem = k - r * T * Cs, s = rem / Cs, c = rem - s * Cs;
      if (MODE == kFwd3) {
        const int ih = reflect(oh[i] + r - 1, H), iw = reflect(ow[i] + s - 1, W);
        return __ldg(a.src + (img + (int64_t)ih * W + iw) * Cs + c);
      } else if (MODE == kFwd2) {
        return __ldg(a.src + (img + (int64_t)(2 * oh[i] + r) * W + 2 * ow[i] + s) * Cs + c);
      } else {
        // dz rows reaching input row ih through tap r: the direct one, and the mirrored border of the padding
        const int ih = oh[i], iw = ow[i];
        const int y0 = ih + 1 - r, y1 = (r == 0 && ih == 1) ? 0 : ((r == 2 && ih == H - 2) ? H - 1 : -1);
        const int x0 = iw + 1 - s, x1 = (s == 0 && iw == 1) ? 0 : ((s == 2 && iw == W - 2) ? W - 1 : -1);
        const int ys[2] = {y0 >= 0 && y0 < H ? y0 : -1, y1};
        const int xs[2] = {x0 >= 0 && x0 < W ? x0 : -1, x1};
        float v = 0.f;
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
          for (int q = 0; q < 2; ++q)
            if (ys[u] >= 0 && xs[q] >= 0) v += __ldg(a.src + (img + (int64_t)ys[u] * W + xs[q]) * Cs + c);
        return v;
      }
    } else {
      return __ldg(a.src + (row0 + row) * (int64_t)K + k);
    }
  };
  auto fb = [&](int, int row, int64_t k) -> float {
    const int n = n0 + row;
    return n < a.N ? __ldg(a.wt + (int64_t)n * K + k) : 0.f;
  };
  float acc[2][4][4];
  gemm_mainloop<false, false>(fa, fb, 0, K, smem, acc);

  // epilogue
  double cs[4][2], cq[4][2];
#pragma unroll
  for (int n = 0; n < 4; ++n) cs[n][0] = cs[n][1] = cq[n][0] = cq[n][1] = 0.0;
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t p = p0 + wm * 32 + m * 16 + g + 8 * h;
      if (p >= P) continue;
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int col = n0 + wn * 32 + n * 8 + 2 * tq + j;
          if (col >= a.N) continue;
          float v = acc[m][n][2 * h + j];
          if (MODE == kFwd3 || MODE == kFwd2 || MODE == kFwd1) {
            v += __ldg(a.bias + col);
            a.out[(b * P + p) * a.N + col] = v;
            cs[n][j] += (double)v;
            cq[n][j] += (double)v * (double)v;
          } else if (MODE == kDgrad2) {
            // col = (r * 2 + s) * Ci + c; dz row (oh, ow) reaches dx pixel (2 oh + r, 2 ow + s) only
            const int Ci = a.N >> 2, rs = col / Ci, c = col - rs * Ci, r = rs >> 1, s = rs & 1;
            const int64_t ohh = p / a.Wo, oww = p - ohh * a.Wo;
            const int64_t ih = 2 * ohh + r, iw = 2 * oww + s;
            const int64_t o = ((b * a.Hx + ih) * a.Wx + iw) * Ci + c;
            a.out[o] = a.add ? v + a.add[o] : v;
            // rows / columns the floor dropped: no tap reaches them
            const bool lr = r == 1 && ohh == a.Ho - 1 && a.Hx > 2 * a.Ho;
            const bool lc = s == 1 && oww == a.Wo - 1 && a.Wx > 2 * a.Wo;
            if (lr) { const int64_t e = o + a.Wx * Ci; a.out[e] = a.add ? a.add[e] : 0.f; }
            if (lc) { const int64_t e = o + Ci; a.out[e] = a.add ? a.add[e] : 0.f; }
            if (lr && lc) { const int64_t e = o + (a.Wx + 1) * Ci; a.out[e] = a.add ? a.add[e] : 0.f; }
          } else {
            const int64_t o = (b * P + p) * a.N + col;
            a.out[o] = a.add ? v + a.add[o] : v;
          }
        }
    }
  if (MODE == kFwd3 || MODE == kFwd2 || MODE == kFwd1) {
    // column sums over the warp's 32 rows (lanes of equal tq), then over the two row halves, then per group
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
        for (int j = 0; j < 2; ++j) colst[wm][wn * 32 + n * 8 + 2 * tq + j] = make_double2(cs[n][j], cq[n][j]);
    }
    __syncthreads();
    const int n_end = min(n0 + BN, a.N);
    const int g_lo = n0 / a.cpg, g_hi = (n_end - 1) / a.cpg;
    const int gg = g_lo + tid;
    if (gg <= g_hi) {
      double s = 0.0, q = 0.0;
      for (int c = max(n0, gg * a.cpg); c < min(n_end, (gg + 1) * a.cpg); ++c) {
        s += colst[0][c - n0].x + colst[1][c - n0].x;
        q += colst[0][c - n0].y + colst[1][c - n0].y;
      }
      a.part[((b * a.tiles + t) * a.ntiles + blockIdx.y) * a.G + gg] = make_double2(s, q);
    }
  }
}

// one CTA per (image, group): mean and invstd from the tile partials, summed in a fixed order
__global__ void __launch_bounds__(kRedThreads)
gn_stats_kernel(const double2* __restrict__ part, int tiles, int ntiles, int G, int cpg, int64_t P, float eps,
                float* __restrict__ mean, float* __restrict__ invstd) {
  __shared__ double sh[kRedThreads];
  const int64_t b = blockIdx.x / G;
  const int gg = (int)(blockIdx.x - b * G);
  const int lo = gg * cpg / BN, hi = ((gg + 1) * cpg - 1) / BN;
  double s = 0.0, q = 0.0;
  for (int t = threadIdx.x; t < tiles; t += kRedThreads)
    for (int nt = lo; nt <= hi; ++nt) {
      const double2 d = part[((b * tiles + t) * ntiles + nt) * G + gg];
      s += d.x;
      q += d.y;
    }
  s = block_sum(s, sh);
  q = block_sum(q, sh);
  if (threadIdx.x == 0) {
    const double n = (double)P * cpg, mu = s / n;
    const double var = fmax(q / n - mu * mu, 0.0);
    mean[blockIdx.x] = (float)mu;
    invstd[blockIdx.x] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

struct WgradArgs {
  const float* dz;    // [B * Ho * Wo, Co]
  const float* x;     // [B * H * W, Ci]
  float* part;        // [splits][Co][Kd + 1]
  int64_t H, W, Ho, Wo, M, rows_per_split;
  int Ci, Co, Kd;
};

// D[oc][j] = sum over the split's output pixels m of dz[m][oc] * im2col(x)[m][j]; j = Kd is a column of ones (dbias)
template <int KIND>
__global__ void __launch_bounds__(kThreads) conv_wgrad_kernel(WgradArgs a) {
  __shared__ __align__(16) float smem[2 * (BM + BN) * LDS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1, g = lane >> 2, tq = lane & 3;
  const int i0 = blockIdx.x * BM, j0 = blockIdx.y * BN;
  const int64_t m_begin = (int64_t)blockIdx.z * a.rows_per_split;
  const int64_t m_end = min(a.M, m_begin + a.rows_per_split);
  const int oc = i0 + (tid & 63), j = j0 + (tid & 63);
  constexpr int T = KIND == DVA_CONV_3X3_REFLECT ? 3 : (KIND == DVA_CONV_2X2_S2 ? 2 : 1);
  const int r = j / (T * a.Ci), rem = j - r * T * a.Ci, s = rem / a.Ci, c = rem - s * a.Ci;
  const int H = (int)a.H, W = (int)a.W;
  const int64_t P = a.Ho * a.Wo;
  auto fa = [&](int, int, int64_t m) -> float { return oc < a.Co ? __ldg(a.dz + m * a.Co + oc) : 0.f; };
  auto fb = [&](int, int, int64_t m) -> float {
    if (j >= a.Kd) return j == a.Kd ? 1.f : 0.f;
    if (KIND == DVA_CONV_1X1) return __ldg(a.x + m * a.Ci + c);
    const int64_t bb = m / P, p = m - bb * P;
    const int oh = (int)(p / a.Wo), ow = (int)(p - (p / a.Wo) * a.Wo);
    const int ih = KIND == DVA_CONV_3X3_REFLECT ? reflect(oh + r - 1, H) : 2 * oh + r;
    const int iw = KIND == DVA_CONV_3X3_REFLECT ? reflect(ow + s - 1, W) : 2 * ow + s;
    return __ldg(a.x + ((bb * H + ih) * W + iw) * a.Ci + c);
  };
  float acc[2][4][4];
  gemm_mainloop<true, true>(fa, fb, m_begin, m_end, smem, acc);
  const int Kp = a.Kd + 1;
  float* out = a.part + (int64_t)blockIdx.z * a.Co * Kp;
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int o = i0 + wm * 32 + m * 16 + g + 8 * h;
      if (o >= a.Co) continue;
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int col = j0 + wn * 32 + n * 8 + 2 * tq + jj;
          if (col < Kp) out[(int64_t)o * Kp + col] = acc[m][n][2 * h + jj];
        }
    }
}

// dwf[oc][j] (j < Kd) and dbias[oc] (j = Kd): the split partials summed in fp64, in split order
__global__ void __launch_bounds__(kRedThreads)
wgrad_reduce_kernel(const float* __restrict__ part, int splits, int Co, int Kd, float* __restrict__ dwf,
                    float* __restrict__ dbias) {
  const int64_t n = (int64_t)Co * (Kd + 1);
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int z = 0; z < splits; ++z) s += (double)part[(int64_t)z * n + e];
    const int oc = (int)(e / (Kd + 1)), j = (int)(e - (int64_t)oc * (Kd + 1));
    if (j < Kd) dwf[(int64_t)oc * Kd + j] = (float)s;
    else dbias[oc] = (float)s;
  }
}

// one CTA per filter oc; w [Co][Ci][T][T] -> wf [Co][T][T][Ci], wd [Ci][T][T][Co] (T = 3, 1) or [T][T][Ci][Co] (T = 2)
__global__ void __launch_bounds__(kRedThreads)
weight_prep_kernel(const float* __restrict__ w, int Co, int Ci, int T, int standardize, float* __restrict__ wf,
                   float* __restrict__ wd) {
  __shared__ double sh[kRedThreads];
  const int oc = blockIdx.x, n = Ci * T * T;
  const float* f = w + (int64_t)oc * n;
  double mu = 0.0, a = 1.0;
  if (standardize) {
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += kRedThreads) s += (double)f[i];
    mu = block_sum(s, sh) / n;
    double q = 0.0;
    for (int i = threadIdx.x; i < n; i += kRedThreads) q += ((double)f[i] - mu) * ((double)f[i] - mu);
    const double sd = sqrt(block_sum(q, sh) / (n - 1));
    a = 1.0 / ((sd + 1e-5) * (double)sqrtf((float)Ci));
  }
  for (int i = threadIdx.x; i < n; i += kRedThreads) {
    const int c = i / (T * T), rs = i - c * T * T;
    const float v = standardize ? (float)(((double)f[i] - mu) * a) : f[i];
    wf[((int64_t)oc * T * T + rs) * Ci + c] = v;
    wd[T == 2 ? ((int64_t)rs * Ci + c) * Co + oc : ((int64_t)c * T * T + rs) * Co + oc] = v;
  }
}

// dw [Co][Ci][T][T] from dwf [Co][T][T][Ci], the gradient of the standardised filter
__global__ void __launch_bounds__(kRedThreads)
weight_prep_bwd_kernel(const float* __restrict__ w, const float* __restrict__ dwf, int Ci, int T,
                       float* __restrict__ dw) {
  __shared__ double sh[kRedThreads];
  const int oc = blockIdx.x, n = Ci * T * T;
  const float* f = w + (int64_t)oc * n;
  const float* gf = dwf + (int64_t)oc * n;
  auto grad = [&](int i) { const int c = i / (T * T), rs = i - c * T * T; return (double)gf[rs * Ci + c]; };
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
  const double a = 1.0 / (den * (double)sqrtf((float)Ci));
  const double k2 = a / den * g2 / ((n - 1) * sd);
  for (int i = threadIdx.x; i < n; i += kRedThreads) {
    const double d = (double)f[i] - mu;
    dw[(int64_t)oc * n + i] = (float)(a * (grad(i) - g1 / n) - k2 * d);
  }
}

__global__ void __launch_bounds__(kRedThreads)
gn_apply_kernel(const float* __restrict__ z, int64_t P, int C, int G, const float* __restrict__ mean,
                const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                float relu_scale, const float* __restrict__ skip, const float* __restrict__ zs,
                const float* __restrict__ mean_s, const float* __restrict__ invstd_s, const float* __restrict__ gamma_s,
                const float* __restrict__ beta_s, float* __restrict__ y, int64_t n) {
  const int cpg = C / G;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / C;
    const int c = (int)(e - row * C);
    const int64_t bg = (row / P) * G + c / cpg;
    float v = (z[e] - mean[bg]) * invstd[bg] * gamma[c] + beta[c];
    if (relu_scale > 0.f) v = fmaxf(v, 0.f) * relu_scale;
    if (skip) v += skip[e];
    if (zs) v += (zs[e] - mean_s[bg]) * invstd_s[bg] * gamma_s[c] + beta_s[c];
    y[e] = v;
  }
}

// the gradient reaching GN(z) and zhat, recomputed from z
struct GnGrad {
  float zh, gu;
};
__device__ __forceinline__ GnGrad gn_grad(float dy, float z, float mu, float is, float ga, float be, float relu_scale) {
  const float zh = (z - mu) * is;
  const float u = zh * ga + be;
  const float gu = relu_scale > 0.f ? (u > 0.f ? dy * relu_scale : 0.f) : dy;
  return {zh, gu};
}

constexpr int kGnRows = 8;   // gn backward CTAs: 32 channels x 8 row lanes

// per (image, chunk of pixels, channel): sums of gu and gu * zhat
__global__ void __launch_bounds__(32 * kGnRows)
gn_bwd_partial_kernel(const float* __restrict__ dy, const float* __restrict__ z, int64_t P, int C, int G,
                      const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                      const float* __restrict__ beta, float relu_scale, int64_t rows_per_chunk,
                      double2* __restrict__ part) {
  __shared__ double2 sh[kGnRows][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.y * 32 + tx;
  const int64_t b = blockIdx.z, chunk = blockIdx.x, chunks = gridDim.x;
  double s1 = 0.0, s2 = 0.0;
  if (c < C) {
    const int64_t bg = b * G + c / (C / G);
    const float mu = mean[bg], is = invstd[bg], ga = gamma[c], be = beta[c];
    const int64_t p_end = min(P, (chunk + 1) * rows_per_chunk);
    for (int64_t p = chunk * rows_per_chunk + ty; p < p_end; p += kGnRows) {
      const int64_t e = (b * P + p) * C + c;
      const GnGrad q = gn_grad(dy[e], z[e], mu, is, ga, be, relu_scale);
      s1 += (double)q.gu;
      s2 += (double)q.gu * (double)q.zh;
    }
  }
  sh[ty][tx] = make_double2(s1, s2);
  __syncthreads();
  if (ty == 0 && c < C) {
    for (int r = 1; r < kGnRows; ++r) {
      s1 += sh[r][tx].x;
      s2 += sh[r][tx].y;
    }
    part[(b * chunks + chunk) * C + c] = make_double2(s1, s2);
  }
}

// per (image, channel): the chunk partials in chunk order
__global__ void __launch_bounds__(32 * kGnRows)
gn_bwd_sums_kernel(const double2* __restrict__ part, int64_t chunks, int C, double2* __restrict__ sums) {
  __shared__ double2 sh[kGnRows][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const int64_t b = blockIdx.y;
  double s1 = 0.0, s2 = 0.0;
  if (c < C)
    for (int64_t k = ty; k < chunks; k += kGnRows) {
      const double2 d = part[(b * chunks + k) * C + c];
      s1 += d.x;
      s2 += d.y;
    }
  sh[ty][tx] = make_double2(s1, s2);
  __syncthreads();
  if (ty == 0 && c < C) {
    for (int r = 1; r < kGnRows; ++r) {
      s1 += sh[r][tx].x;
      s2 += sh[r][tx].y;
    }
    sums[b * C + c] = make_double2(s1, s2);
  }
}

// dbeta, dgamma per channel (sum over images) and the per-(image, group) means of gamma * gu and gamma * gu * zhat
__global__ void __launch_bounds__(kRedThreads)
gn_bwd_coef_kernel(const double2* __restrict__ sums, int64_t B, int64_t P, int C, int G,
                   const float* __restrict__ gamma, float* __restrict__ dgamma, float* __restrict__ dbeta,
                   double2* __restrict__ coef) {
  const int cpg = C / G;
  for (int c = threadIdx.x; c < C; c += kRedThreads) {
    double s1 = 0.0, s2 = 0.0;
    for (int64_t b = 0; b < B; ++b) {
      s1 += sums[b * C + c].x;
      s2 += sums[b * C + c].y;
    }
    dbeta[c] = (float)s1;
    dgamma[c] = (float)s2;
  }
  const double n = (double)P * cpg;
  for (int64_t bg = threadIdx.x; bg < B * G; bg += kRedThreads) {
    const int64_t b = bg / G;
    const int gg = (int)(bg - b * G);
    double s1 = 0.0, s2 = 0.0;
    for (int c = gg * cpg; c < (gg + 1) * cpg; ++c) {
      s1 += (double)gamma[c] * sums[b * C + c].x;
      s2 += (double)gamma[c] * sums[b * C + c].y;
    }
    coef[bg] = make_double2(s1 / n, s2 / n);
  }
}

__global__ void __launch_bounds__(kRedThreads)
gn_bwd_dz_kernel(const float* __restrict__ dy, const float* __restrict__ z, int64_t P, int C, int G,
                 const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float relu_scale, const double2* __restrict__ coef,
                 float* __restrict__ dz, int64_t n) {
  const int cpg = C / G;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / C;
    const int c = (int)(e - row * C);
    const int64_t bg = (row / P) * G + c / cpg;
    const float is = invstd[bg];
    const GnGrad q = gn_grad(dy[e], z[e], mean[bg], is, gamma[c], beta[c], relu_scale);
    const double2 k = coef[bg];
    dz[e] = (float)((double)is * ((double)q.gu * gamma[c] - k.x - (double)q.zh * k.y));
  }
}

// ---- host-side sizes
inline int64_t out_size(int kind, int64_t n) { return kind == DVA_CONV_2X2_S2 ? n / 2 : n; }
inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

inline int check_shape(const char* what, int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind) {
  if (kind != DVA_CONV_3X3_REFLECT && kind != DVA_CONV_2X2_S2 && kind != DVA_CONV_1X1)
    return failf(DVA_EINVAL, "%s: unknown kind", what);
  if (B < 1 || H < 1 || W < 1 || Ci < 1 || Co < 1) return failf(DVA_EINVAL, "%s: bad sizes", what);
  if (kind != DVA_CONV_1X1 && (H < 2 || W < 2))
    return failf(DVA_EINVAL, "%s: every spatial side must be >= 2 (got %lld x %lld)", what, (long long)H,
                 (long long)W);
  const int64_t T = taps_of(kind);
  if ((int64_t)Co * T * T * Ci > (int64_t)INT32_MAX / 4 || H > INT32_MAX / 2 || W > INT32_MAX / 2)
    return failf(DVA_EUNSUPPORTED, "%s: sizes beyond the 32-bit index range", what);
  return DVA_OK;
}

struct FwdPlan {
  int64_t Ho, Wo, P;
  int tiles, ntiles;
};
inline FwdPlan fwd_plan(int64_t H, int64_t W, int Co, int kind) {
  FwdPlan p;
  p.Ho = out_size(kind, H);
  p.Wo = out_size(kind, W);
  p.P = p.Ho * p.Wo;
  p.tiles = (int)cdiv(p.P, BM);
  p.ntiles = (int)cdiv(Co, BN);
  return p;
}

struct WgradPlan {
  int64_t M, rows_per_split;
  int splits, Kd;
};
inline WgradPlan wgrad_plan(int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind) {
  WgradPlan p;
  const int T = taps_of(kind);
  p.M = B * out_size(kind, H) * out_size(kind, W);
  p.Kd = T * T * Ci;
  const int64_t tiles_mn = cdiv(Co, BM) * cdiv(p.Kd + 1, BN);
  const int64_t want = std::max<int64_t>(1, cdiv(4 * kNumSMs, tiles_mn));
  const int64_t splits = std::min<int64_t>(want, cdiv(p.M, 4 * BK));
  p.rows_per_split = cdiv(cdiv(p.M, splits), BK) * BK;
  p.splits = (int)cdiv(p.M, p.rows_per_split);
  return p;
}

struct GnPlan {
  int64_t chunks, rows_per_chunk;
};
inline GnPlan gn_plan(int64_t B, int64_t P, int C) {
  GnPlan p;
  const int64_t cap = std::max<int64_t>(1, 1024 / (B * cdiv(C, 32)));
  p.chunks = std::max<int64_t>(1, std::min<int64_t>(cdiv(P, 256), cap));
  p.rows_per_chunk = cdiv(P, p.chunks);
  p.chunks = cdiv(P, p.rows_per_chunk);
  return p;
}

template <int MODE> int launch_gemm(const GemmArgs& a, int64_t B, cudaStream_t st, const char* what) {
  const dim3 grid((unsigned)(B * a.tiles), (unsigned)cdiv(a.N, BN));
  conv_gemm_kernel<MODE><<<grid, kThreads, 0, st>>>(a);
  return check_launch(what);
}

inline int elementwise_grid(int64_t n) { return grid_cap(n, kRedThreads, 8); }

}  // namespace dva_conv2d

using namespace dva;
using namespace dva_conv2d;

extern "C" int dva_conv2d_weight_prep(const float* w, int Co, int Ci, int kind, int standardize, float* wf, float* wd,
                                      void* stream) {
  const int rc = check_shape("conv2d_weight_prep", 1, 2, 2, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (!w || !wf || !wd) return fail(DVA_EINVAL, "conv2d_weight_prep: null pointer");
  if (standardize && Ci * taps_of(kind) * taps_of(kind) < 2)
    return fail(DVA_EINVAL, "conv2d_weight_prep: standardisation needs at least 2 weights per filter");
  weight_prep_kernel<<<Co, kRedThreads, 0, (cudaStream_t)stream>>>(w, Co, Ci, taps_of(kind), standardize, wf, wd);
  return check_launch("conv2d_weight_prep");
}

extern "C" int dva_conv2d_weight_prep_bwd(const float* w, const float* dwf, int Co, int Ci, int kind, float* dw,
                                          void* stream) {
  const int rc = check_shape("conv2d_weight_prep_bwd", 1, 2, 2, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (!w || !dwf || !dw) return fail(DVA_EINVAL, "conv2d_weight_prep_bwd: null pointer");
  if (Ci * taps_of(kind) * taps_of(kind) < 2)
    return fail(DVA_EINVAL, "conv2d_weight_prep_bwd: standardisation needs at least 2 weights per filter");
  weight_prep_bwd_kernel<<<Co, kRedThreads, 0, (cudaStream_t)stream>>>(w, dwf, Ci, taps_of(kind), dw);
  return check_launch("conv2d_weight_prep_bwd");
}

extern "C" size_t dva_conv2d_fwd_workspace_bytes(int64_t B, int64_t Ho, int64_t Wo, int Co, int G) {
  if (B < 1 || Ho < 1 || Wo < 1 || Co < 1 || G < 1) return 0;
  return (size_t)B * cdiv(Ho * Wo, BM) * cdiv(Co, BN) * G * sizeof(double2);
}

extern "C" int dva_conv2d_fwd(const float* x, int64_t B, int64_t H, int64_t W, int Ci, const float* wf,
                              const float* bias, int Co, int kind, int G, float eps, float* z, float* mean,
                              float* invstd, void* ws, size_t ws_bytes, void* stream) {
  const int rc = check_shape("conv2d_fwd", B, H, W, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (G < 1 || Co % G != 0) return fail(DVA_EINVAL, "conv2d_fwd: the groups must divide the channels");
  if (!x || !wf || !bias || !z || !mean || !invstd || !ws) return fail(DVA_EINVAL, "conv2d_fwd: null pointer");
  const FwdPlan pl = fwd_plan(H, W, Co, kind);
  if (ws_bytes < dva_conv2d_fwd_workspace_bytes(B, pl.Ho, pl.Wo, Co, G))
    return fail(DVA_EINVAL, "conv2d_fwd: workspace too small");
  if (B * pl.tiles > INT32_MAX) return fail(DVA_EUNSUPPORTED, "conv2d_fwd: too many pixels");
  const int T = taps_of(kind);
  GemmArgs a{};
  a.src = x; a.wt = wf; a.bias = bias; a.out = z; a.part = (double2*)ws;
  a.H = H; a.W = W; a.Ho = pl.Ho; a.Wo = pl.Wo; a.Cs = Ci; a.N = Co; a.K = T * T * Ci;
  a.G = G; a.cpg = Co / G; a.tiles = pl.tiles; a.ntiles = pl.ntiles;
  cudaStream_t st = (cudaStream_t)stream;
  int r2 = kind == DVA_CONV_3X3_REFLECT ? launch_gemm<kFwd3>(a, B, st, "conv2d_fwd")
         : kind == DVA_CONV_2X2_S2     ? launch_gemm<kFwd2>(a, B, st, "conv2d_fwd")
                                       : launch_gemm<kFwd1>(a, B, st, "conv2d_fwd");
  if (r2 != DVA_OK) return r2;
  gn_stats_kernel<<<(unsigned)(B * G), kRedThreads, 0, st>>>(a.part, pl.tiles, pl.ntiles, G, Co / G, pl.P, eps,
                                                             mean, invstd);
  return check_launch("conv2d_fwd_stats");
}

extern "C" int dva_conv2d_dgrad(const float* dz, int64_t B, int64_t H, int64_t W, int Ci, int Co, const float* wd,
                                int kind, const float* add, float* dx, void* stream) {
  const int rc = check_shape("conv2d_dgrad", B, H, W, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (!dz || !wd || !dx) return fail(DVA_EINVAL, "conv2d_dgrad: null pointer");
  GemmArgs a{};
  a.src = dz; a.wt = wd; a.add = add; a.out = dx; a.H = H; a.W = W; a.Cs = Co;
  cudaStream_t st = (cudaStream_t)stream;
  if (kind == DVA_CONV_2X2_S2) {
    a.Ho = H / 2; a.Wo = W / 2; a.Hx = H; a.Wx = W; a.N = 4 * Ci; a.K = Co;
  } else {
    a.Ho = H; a.Wo = W; a.N = Ci; a.K = taps_of(kind) * taps_of(kind) * Co;
  }
  a.tiles = (int)cdiv(a.Ho * a.Wo, BM);
  if (B * a.tiles > INT32_MAX) return fail(DVA_EUNSUPPORTED, "conv2d_dgrad: too many pixels");
  return kind == DVA_CONV_3X3_REFLECT ? launch_gemm<kDgrad3>(a, B, st, "conv2d_dgrad")
       : kind == DVA_CONV_2X2_S2     ? launch_gemm<kDgrad2>(a, B, st, "conv2d_dgrad")
                                     : launch_gemm<kDgrad1>(a, B, st, "conv2d_dgrad");
}

extern "C" size_t dva_conv2d_wgrad_workspace_bytes(int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind) {
  if (B < 1 || H < 1 || W < 1 || Ci < 1 || Co < 1 || taps_of(kind) < 1) return 0;
  if (kind != DVA_CONV_1X1 && (H < 2 || W < 2)) return 0;
  const WgradPlan p = wgrad_plan(B, H, W, Ci, Co, kind);
  return (size_t)p.splits * Co * (p.Kd + 1) * sizeof(float);
}

extern "C" int dva_conv2d_wgrad(const float* dz, const float* x, int64_t B, int64_t H, int64_t W, int Ci, int Co,
                                int kind, float* dwf, float* dbias, void* ws, size_t ws_bytes, void* stream) {
  const int rc = check_shape("conv2d_wgrad", B, H, W, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (!dz || !x || !dwf || !dbias || !ws) return fail(DVA_EINVAL, "conv2d_wgrad: null pointer");
  if (ws_bytes < dva_conv2d_wgrad_workspace_bytes(B, H, W, Ci, Co, kind))
    return fail(DVA_EINVAL, "conv2d_wgrad: workspace too small");
  const WgradPlan pl = wgrad_plan(B, H, W, Ci, Co, kind);
  WgradArgs a{};
  a.dz = dz; a.x = x; a.part = (float*)ws;
  a.H = H; a.W = W; a.Ho = out_size(kind, H); a.Wo = out_size(kind, W); a.M = pl.M;
  a.rows_per_split = pl.rows_per_split; a.Ci = Ci; a.Co = Co; a.Kd = pl.Kd;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)cdiv(Co, BM), (unsigned)cdiv(pl.Kd + 1, BN), (unsigned)pl.splits);
  if (kind == DVA_CONV_3X3_REFLECT) conv_wgrad_kernel<DVA_CONV_3X3_REFLECT><<<grid, kThreads, 0, st>>>(a);
  else if (kind == DVA_CONV_2X2_S2) conv_wgrad_kernel<DVA_CONV_2X2_S2><<<grid, kThreads, 0, st>>>(a);
  else conv_wgrad_kernel<DVA_CONV_1X1><<<grid, kThreads, 0, st>>>(a);
  const int r2 = check_launch("conv2d_wgrad");
  if (r2 != DVA_OK) return r2;
  wgrad_reduce_kernel<<<elementwise_grid((int64_t)Co * (pl.Kd + 1)), kRedThreads, 0, st>>>(a.part, pl.splits, Co,
                                                                                           pl.Kd, dwf, dbias);
  return check_launch("conv2d_wgrad_reduce");
}

extern "C" int dva_conv2d_gn_apply(const float* z, int64_t B, int64_t P, int C, int G, const float* mean,
                                   const float* invstd, const float* gamma, const float* beta, float relu_scale,
                                   const float* skip, const float* zs, const float* mean_s, const float* invstd_s,
                                   const float* gamma_s, const float* beta_s, float* y, void* stream) {
  if (B < 1 || P < 1 || C < 1 || G < 1 || C % G != 0) return fail(DVA_EINVAL, "conv2d_gn_apply: bad sizes");
  if (relu_scale < 0.f) return fail(DVA_EINVAL, "conv2d_gn_apply: negative relu_scale");
  if (!z || !mean || !invstd || !gamma || !beta || !y) return fail(DVA_EINVAL, "conv2d_gn_apply: null pointer");
  if (zs && (!mean_s || !invstd_s || !gamma_s || !beta_s)) return fail(DVA_EINVAL, "conv2d_gn_apply: null pointer");
  const int64_t n = B * P * C;
  gn_apply_kernel<<<elementwise_grid(n), kRedThreads, 0, (cudaStream_t)stream>>>(
      z, P, C, G, mean, invstd, gamma, beta, relu_scale, skip, zs, mean_s, invstd_s, gamma_s, beta_s, y, n);
  return check_launch("conv2d_gn_apply");
}

extern "C" size_t dva_conv2d_gn_bwd_workspace_bytes(int64_t B, int64_t P, int C, int G) {
  if (B < 1 || P < 1 || C < 1 || G < 1) return 0;
  const GnPlan p = gn_plan(B, P, C);
  return round256((size_t)B * p.chunks * C * sizeof(double2)) + round256((size_t)B * C * sizeof(double2)) +
         (size_t)B * G * sizeof(double2);
}

extern "C" int dva_conv2d_gn_bwd(const float* dy, const float* z, int64_t B, int64_t P, int C, int G,
                                 const float* mean, const float* invstd, const float* gamma, const float* beta,
                                 float relu_scale, float* dz, float* dgamma, float* dbeta, void* ws, size_t ws_bytes,
                                 void* stream) {
  if (B < 1 || P < 1 || C < 1 || G < 1 || C % G != 0) return fail(DVA_EINVAL, "conv2d_gn_bwd: bad sizes");
  if (relu_scale < 0.f) return fail(DVA_EINVAL, "conv2d_gn_bwd: negative relu_scale");
  if (!dy || !z || !mean || !invstd || !gamma || !beta || !dz || !dgamma || !dbeta || !ws)
    return fail(DVA_EINVAL, "conv2d_gn_bwd: null pointer");
  if (ws_bytes < dva_conv2d_gn_bwd_workspace_bytes(B, P, C, G))
    return fail(DVA_EINVAL, "conv2d_gn_bwd: workspace too small");
  if (B > 65535) return fail(DVA_EUNSUPPORTED, "conv2d_gn_bwd: more than 65535 images");
  const GnPlan pl = gn_plan(B, P, C);
  uint8_t* base = (uint8_t*)ws;
  double2* part = (double2*)base;
  double2* sums = (double2*)(base + round256((size_t)B * pl.chunks * C * sizeof(double2)));
  double2* coef = (double2*)((uint8_t*)sums + round256((size_t)B * C * sizeof(double2)));
  cudaStream_t st = (cudaStream_t)stream;
  const int cb = (int)cdiv(C, 32);
  gn_bwd_partial_kernel<<<dim3((unsigned)pl.chunks, cb, (unsigned)B), 32 * kGnRows, 0, st>>>(
      dy, z, P, C, G, mean, invstd, gamma, beta, relu_scale, pl.rows_per_chunk, part);
  int rc = check_launch("conv2d_gn_bwd_partial");
  if (rc != DVA_OK) return rc;
  gn_bwd_sums_kernel<<<dim3(cb, (unsigned)B), 32 * kGnRows, 0, st>>>(part, pl.chunks, C, sums);
  rc = check_launch("conv2d_gn_bwd_sums");
  if (rc != DVA_OK) return rc;
  gn_bwd_coef_kernel<<<1, kRedThreads, 0, st>>>(sums, B, P, C, G, gamma, dgamma, dbeta, coef);
  rc = check_launch("conv2d_gn_bwd_coef");
  if (rc != DVA_OK) return rc;
  const int64_t n = B * P * C;
  gn_bwd_dz_kernel<<<elementwise_grid(n), kRedThreads, 0, st>>>(dy, z, P, C, G, mean, invstd, gamma, beta,
                                                                relu_scale, coef, dz, n);
  return check_launch("conv2d_gn_bwd_dz");
}
