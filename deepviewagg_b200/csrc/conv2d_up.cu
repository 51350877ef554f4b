// The from-scratch image decoder (libdva_unet.so, C ABI include/dva_unet.h): weight-standardised transposed
// convolutions (ConvTranspose2dWS of ResNetUp) with the GroupNorm statistics in their epilogue.
//
//   convt_weight_prep_kernel / convt_weight_prep_bwd_kernel  one CTA per input channel c of w [Ci][Co][R][S]:
//        mean and unbiased std over Co*R*S in fp64, divided by sqrt(Co) taken in fp32 (standardize_weights of
//        image.py:39-50 on a transposed weight); writes the filters the GEMMs read, and maps the gradient of the
//        forward's filter back to the torch layout.
//   convt_gemm_kernel<MODE>  the main loop of conv2d_gemm.cuh (64 x 64 tiles, mma.sync in 3xTF32):
//          kUp2      rows of x against [R][S][Co] x Ci: [B*H*W, Ci] x [Ci, 4 Co]; the epilogue adds the bias and
//                    scatters column group (a, b) of pixel (i, j) to pixel (2i + a, 2j + b)
//          kFwdT3    3x3 zero-padded taps of x against the flipped filter
//          kDgradT3  3x3 zero-padded taps of dz against the unflipped filter
//          kDgradUp2 2x2 stride-2 taps of dz (the transposed 2x2 has no floor: every dz pixel is read once)
//        The forward epilogues take per-column fp64 sums of z and z^2 and reduce them to one partial per (tile,
//        column tile, group); a tile never straddles two images.
//   convt_stats_kernel  one CTA per (image, group): the partials in a fixed order -> mean, invstd.
//   convt_wgrad_kernel<KIND> + convt_wgrad_reduce_kernel  the gradient of the forward's filter split over the
//        pixels, one fp32 partial per split, summed in fp64 in split order; a column of ones gives dbias (for
//        kUp2 one sum per (a, b, o), folded over (a, b) in the reduction).
//   unary_act_kernel / unary_act_bwd_kernel  relu(z) * scale and its backward (UnaryConv's activation).
// GroupNorm apply / backward, ReLUWS, the residual and the 1x1 convolutions are those of libdva_conv2d.so.
// Nothing that is summed uses atomics: every result is bitwise reproducible run to run.
#include "dva_common.cuh"
#include "../../include/dva_unet.h"
#include "conv2d_gemm.cuh"
#include <algorithm>

// namespace dva_unet: the kernels of libdva_unet.so (case table: tests/test_unet_matrix_table.py)
namespace dva_unet {
using namespace dva;
using namespace dva_convgemm;

enum { kUp2 = 0, kFwdT3 = 1, kDgradT3 = 2, kDgradUp2 = 3 };

__host__ __device__ __forceinline__ int taps_of(int kind) { return kind == DVA_UNET_UP_2X2 ? 2 : 3; }

struct ConvTArgs {
  const float* src;   // the gathered operand: x (forward) or dz (data gradient)
  const float* wt;    // [N][K]
  const float* bias;  // forward
  const float* add;   // data gradient: out = acc + add
  float* out;
  double2* part;      // forward: one (sum, sum of squares) per (tile, column tile, group)
  int64_t H, W;       // spatial size of src
  int64_t Ho, Wo;     // the grid of GEMM rows, per image (P = Ho * Wo)
  int Cs;             // channels of src
  int N, K;
  int Cg;             // forward: output channels; the group of column n is (n % Cg) / cpg
  int G, cpg, tiles, ntiles;
};

template <int MODE>
__global__ void __launch_bounds__(kThreads) convt_gemm_kernel(ConvTArgs a) {
  __shared__ __align__(16) float smem[2 * (BM + BN) * LDS];
  __shared__ double2 colst[2][BN];
  constexpr bool kFwd = MODE == kUp2 || MODE == kFwdT3;
  const int tid = threadIdx.x;
  const int64_t b = blockIdx.x / a.tiles;
  const int t = (int)(blockIdx.x - b * a.tiles);
  const int64_t P = a.Ho * a.Wo, p0 = (int64_t)t * BM;
  const int n0 = blockIdx.y * BN;
  const int64_t img = b * a.H * a.W;   // first source pixel of image b
  const int64_t row0 = b * P + p0;     // first GEMM row of the tile
  int oh[8], ow[8];
  tile_pixels(p0, P, a.Wo, oh, ow);
  const int H = (int)a.H, W = (int)a.W, Cs = a.Cs, K = a.K;
  auto fa = [&](int i, int row, int64_t k64) -> float {
    if (oh[i] < 0) return 0.f;
    const int k = (int)k64;
    if (MODE == kUp2) return __ldg(a.src + (row0 + row) * (int64_t)K + k);
    const int T = MODE == kDgradUp2 ? 2 : 3;
    const int r = k / (T * Cs), rem = k - r * T * Cs, s = rem / Cs, c = rem - s * Cs;
    if (MODE == kDgradUp2) return __ldg(a.src + (img + (int64_t)(2 * oh[i] + r) * W + 2 * ow[i] + s) * Cs + c);
    const int ih = oh[i] + r - 1, iw = ow[i] + s - 1;
    if (ih < 0 || ih >= H || iw < 0 || iw >= W) return 0.f;
    return __ldg(a.src + (img + (int64_t)ih * W + iw) * Cs + c);
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
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int64_t p = p0 + acc_row(m, q);
        const int col = n0 + acc_col(n, q);
        if (p >= P || col >= a.N) continue;
        float v = acc[m][n][q];
        int64_t o;
        if (MODE == kUp2) {
          // col = (r * 2 + s) * Co + c: pixel (oh, ow) of x reaches pixel (2 oh + r, 2 ow + s) of z
          const int Co = a.Cg, rs = col / Co, c = col - rs * Co;
          const int64_t ohh = p / a.Wo, oww = p - ohh * a.Wo;
          v += __ldg(a.bias + c);
          o = ((b * 2 * a.Ho + 2 * ohh + (rs >> 1)) * 2 * a.Wo + 2 * oww + (rs & 1)) * Co + c;
        } else {
          o = (b * P + p) * a.N + col;
          if (MODE == kFwdT3) v += __ldg(a.bias + col);
          else if (a.add) v += a.add[o];
        }
        a.out[o] = v;
        if (kFwd) {
          cs[n][q & 1] += (double)v;
          cq[n][q & 1] += (double)v * (double)v;
        }
      }
  if (kFwd) {
    // column sums over the two row halves, then per group
    column_stats(cs, cq, colst);
    // every group gets a partial (0 where the column tile has none of its columns): with kUp2 a column tile can
    // wrap around the channels
    if (tid < a.G) {
      double s = 0.0, q = 0.0;
      for (int c = n0; c < min(n0 + BN, a.N); ++c)
        if ((c % a.Cg) / a.cpg == tid) {
          s += colst[0][c - n0].x + colst[1][c - n0].x;
          q += colst[0][c - n0].y + colst[1][c - n0].y;
        }
      a.part[((b * a.tiles + t) * a.ntiles + blockIdx.y) * a.G + tid] = make_double2(s, q);
    }
  }
}

// one CTA per (image, group): mean and invstd from the (tile, column tile) partials, summed in a fixed order
__global__ void __launch_bounds__(kRedThreads)
convt_stats_kernel(const double2* __restrict__ part, int tiles, int ntiles, int G, int64_t n_group, float eps,
                   float* __restrict__ mean, float* __restrict__ invstd) {
  __shared__ double sh[kRedThreads];
  const int64_t b = blockIdx.x / G;
  const int gg = (int)(blockIdx.x - b * G);
  double s = 0.0, q = 0.0;
  for (int t = threadIdx.x; t < tiles; t += kRedThreads)
    for (int nt = 0; nt < ntiles; ++nt) {
      const double2 d = part[((b * tiles + t) * ntiles + nt) * G + gg];
      s += d.x;
      q += d.y;
    }
  finish_stats(s, q, (double)n_group, eps, mean[blockIdx.x], invstd[blockIdx.x], sh);
}

struct ConvTWgradArgs {
  const float* dz;    // [B * H' * W', Co]
  const float* x;     // [B * H * W, Ci]
  float* part;        // [splits][Rw][Kd + 1]
  int64_t H, W, M, rows_per_split;
  int Ci, Co, Rw, Kd;
};

// D[r][j] = sum over the split's pixels m of A[m][r] * X[m][j], j = Kd a column of ones (dbias):
//   DVA_UNET_T_3X3   r = o, m over the output pixels, X = the zero-padded taps of x, j = (ky * 3 + kx) * Ci + c
//   DVA_UNET_UP_2X2  r = (a * 2 + b) * Co + o, m over the pixels (i, j) of x, A[m][r] = dz at (2i + a, 2j + b)
template <int KIND>
__global__ void __launch_bounds__(kThreads) convt_wgrad_kernel(ConvTWgradArgs a) {
  __shared__ __align__(16) float smem[2 * (BM + BN) * LDS];
  const int i0 = blockIdx.x * BM, j0 = blockIdx.y * BN;
  const int64_t m_begin = (int64_t)blockIdx.z * a.rows_per_split;
  const int64_t m_end = min(a.M, m_begin + a.rows_per_split);
  const int rr = i0 + (threadIdx.x & 63), j = j0 + (threadIdx.x & 63);
  const int H = (int)a.H, W = (int)a.W;
  const int64_t P = a.H * a.W;
  const int ab = KIND == DVA_UNET_UP_2X2 ? rr / a.Co : 0, oc = rr - ab * a.Co;
  const int r = j / (3 * a.Ci), rem = j - r * 3 * a.Ci, s = rem / a.Ci, c = rem - s * a.Ci;
  auto fa = [&](int, int, int64_t m) -> float {
    if (rr >= a.Rw) return 0.f;
    if (KIND == DVA_UNET_T_3X3) return __ldg(a.dz + m * a.Co + oc);
    const int64_t bb = m / P, p = m - bb * P;
    const int ih = (int)(p / W), iw = (int)(p - (p / W) * W);
    return __ldg(a.dz + ((bb * 2 * H + 2 * ih + (ab >> 1)) * 2 * W + 2 * iw + (ab & 1)) * a.Co + oc);
  };
  auto fb = [&](int, int, int64_t m) -> float {
    if (j >= a.Kd) return j == a.Kd ? 1.f : 0.f;
    if (KIND == DVA_UNET_UP_2X2) return __ldg(a.x + m * a.Ci + j);
    const int64_t bb = m / P, p = m - bb * P;
    const int ih = (int)(p / W) + r - 1, iw = (int)(p - (p / W) * W) + s - 1;
    if (ih < 0 || ih >= H || iw < 0 || iw >= W) return 0.f;
    return __ldg(a.x + ((bb * H + ih) * W + iw) * a.Ci + c);
  };
  float acc[2][4][4];
  gemm_mainloop<true, true>(fa, fb, m_begin, m_end, smem, acc);
  const int Kp = a.Kd + 1;
  store_tile(acc, i0, j0, a.Rw, Kp, Kp, a.part + (int64_t)blockIdx.z * a.Rw * Kp);
}

// dwf [Rw][Kd] and dbias [Co]: the split partials summed in fp64, in split order; dbias folds the Rw / Co
// column-of-ones sums of channel o in (a, b) order
__global__ void __launch_bounds__(kRedThreads)
convt_wgrad_reduce_kernel(const float* __restrict__ part, int splits, int Rw, int Kd, int Co,
                          float* __restrict__ dwf, float* __restrict__ dbias) {
  const int64_t Kp = Kd + 1, per_split = (int64_t)Rw * Kp, nw = (int64_t)Rw * Kd, fold = Rw / Co;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nw + Co;
       e += (int64_t)gridDim.x * blockDim.x) {
    double s = 0.0;
    if (e < nw) {
      const int64_t r = e / Kd, j = e - r * Kd;
      for (int z = 0; z < splits; ++z) s += (double)part[z * per_split + r * Kp + j];
      dwf[e] = (float)s;
    } else {
      const int64_t o = e - nw;
      for (int64_t f = 0; f < fold; ++f)
        for (int z = 0; z < splits; ++z) s += (double)part[z * per_split + (f * Co + o) * Kp + Kd];
      dbias[o] = (float)s;
    }
  }
}

// where element i = o * T * T + rs of input channel c's filter goes in wf (the forward's operand) and wd (the data
// gradient's)
__device__ __forceinline__ int64_t wf_index(int c, int o, int rs, int Ci, int Co, int T) {
  return T == 2 ? ((int64_t)rs * Co + o) * Ci + c : ((int64_t)o * 9 + (8 - rs)) * Ci + c;
}

// one CTA per input channel c; w [Ci][Co][T][T] -> wf, wd (include/dva_unet.h)
__global__ void __launch_bounds__(kRedThreads)
convt_weight_prep_kernel(const float* __restrict__ w, int Ci, int Co, int T, float* __restrict__ wf,
                         float* __restrict__ wd) {
  __shared__ double sh[kRedThreads];
  const int c = blockIdx.x, n = Co * T * T;
  standardize_filter(w + (int64_t)c * n, n, Co, sh, [&](int i, float v) {
    const int o = i / (T * T), rs = i - o * T * T;
    wf[wf_index(c, o, rs, Ci, Co, T)] = v;
    wd[((int64_t)c * T * T + rs) * Co + o] = v;
  });
}

// dw [Ci][Co][T][T] from dwf (the layout of wf), the gradient of the standardised filter
__global__ void __launch_bounds__(kRedThreads)
convt_weight_prep_bwd_kernel(const float* __restrict__ w, const float* __restrict__ dwf, int Ci, int Co, int T,
                             float* __restrict__ dw) {
  __shared__ double sh[kRedThreads];
  const int c = blockIdx.x, n = Co * T * T;
  auto grad = [&](int i) { const int o = i / (T * T), rs = i - o * T * T; return (double)dwf[wf_index(c, o, rs, Ci, Co, T)]; };
  standardize_filter_bwd(w + (int64_t)c * n, n, Co, sh, grad, dw + (int64_t)c * n);
}

__global__ void __launch_bounds__(kRedThreads)
unary_act_kernel(const float* __restrict__ z, int64_t n, float scale, float* __restrict__ y) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
    y[e] = fmaxf(z[e], 0.f) * scale;
}

__global__ void __launch_bounds__(kRedThreads)
unary_act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ z, int64_t n, float scale,
                     float* __restrict__ dz) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
    dz[e] = z[e] > 0.f ? dy[e] * scale : 0.f;
}

// ---- host-side sizes
inline int check_shape(const char* what, int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind) {
  if (kind != DVA_UNET_UP_2X2 && kind != DVA_UNET_T_3X3) return failf(DVA_EINVAL, "%s: unknown kind", what);
  if (B < 1 || H < 1 || W < 1 || Ci < 1 || Co < 1) return failf(DVA_EINVAL, "%s: bad sizes", what);
  const int64_t T = taps_of(kind);
  if ((int64_t)Co * T * T * Ci > (int64_t)INT32_MAX / 4 || H > INT32_MAX / 4 || W > INT32_MAX / 4)
    return failf(DVA_EUNSUPPORTED, "%s: sizes beyond the 32-bit index range", what);
  return DVA_OK;
}

struct WgradPlan {
  int64_t M, rows_per_split;
  int splits, Rw, Kd;
};
inline WgradPlan wgrad_plan(int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind) {
  WgradPlan p;
  p.M = B * H * W;
  p.Rw = kind == DVA_UNET_UP_2X2 ? 4 * Co : Co;
  p.Kd = kind == DVA_UNET_UP_2X2 ? Ci : 9 * Ci;
  const SplitRows s = split_rows(p.M, cdiv(p.Rw, BM) * cdiv(p.Kd + 1, BN));
  p.rows_per_split = s.rows_per_split;
  p.splits = s.splits;
  return p;
}

template <int MODE> int launch_gemm(const ConvTArgs& a, int64_t B, cudaStream_t st, const char* what) {
  const dim3 grid((unsigned)(B * a.tiles), (unsigned)cdiv(a.N, BN));
  convt_gemm_kernel<MODE><<<grid, kThreads, 0, st>>>(a);
  return check_launch(what);
}

}  // namespace dva_unet

using namespace dva;
using namespace dva_unet;

extern "C" int dva_unet_weight_prep(const float* w, int Ci, int Co, int kind, float* wf, float* wd, void* stream) {
  const int rc = check_shape("unet_weight_prep", 1, 1, 1, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (!w || !wf || !wd) return fail(DVA_EINVAL, "unet_weight_prep: null pointer");
  convt_weight_prep_kernel<<<Ci, kRedThreads, 0, (cudaStream_t)stream>>>(w, Ci, Co, taps_of(kind), wf, wd);
  return check_launch("unet_weight_prep");
}

extern "C" int dva_unet_weight_prep_bwd(const float* w, const float* dwf, int Ci, int Co, int kind, float* dw,
                                        void* stream) {
  const int rc = check_shape("unet_weight_prep_bwd", 1, 1, 1, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (!w || !dwf || !dw) return fail(DVA_EINVAL, "unet_weight_prep_bwd: null pointer");
  convt_weight_prep_bwd_kernel<<<Ci, kRedThreads, 0, (cudaStream_t)stream>>>(w, dwf, Ci, Co, taps_of(kind), dw);
  return check_launch("unet_weight_prep_bwd");
}

extern "C" size_t dva_unet_fwd_workspace_bytes(int64_t B, int64_t H, int64_t W, int Co, int G, int kind) {
  if (B < 1 || H < 1 || W < 1 || Co < 1 || G < 1 || (kind != DVA_UNET_UP_2X2 && kind != DVA_UNET_T_3X3)) return 0;
  const int N = kind == DVA_UNET_UP_2X2 ? 4 * Co : Co;
  return (size_t)B * cdiv(H * W, BM) * cdiv(N, BN) * G * sizeof(double2);
}

extern "C" int dva_unet_fwd(const float* x, int64_t B, int64_t H, int64_t W, int Ci, const float* wf,
                            const float* bias, int Co, int kind, int G, float eps, float* z, float* mean,
                            float* invstd, void* ws, size_t ws_bytes, void* stream) {
  const int rc = check_shape("unet_fwd", B, H, W, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (G < 1 || Co % G != 0) return fail(DVA_EINVAL, "unet_fwd: the groups must divide the channels");
  if (G > kThreads) return failf(DVA_EUNSUPPORTED, "unet_fwd: at most %d groups", kThreads);
  if (!x || !wf || !bias || !z || !mean || !invstd || !ws) return fail(DVA_EINVAL, "unet_fwd: null pointer");
  if (ws_bytes < dva_unet_fwd_workspace_bytes(B, H, W, Co, G, kind))
    return fail(DVA_EINVAL, "unet_fwd: workspace too small");
  const bool up = kind == DVA_UNET_UP_2X2;
  ConvTArgs a{};
  a.src = x; a.wt = wf; a.bias = bias; a.out = z; a.part = (double2*)ws;
  a.H = H; a.W = W; a.Ho = H; a.Wo = W; a.Cs = Ci;
  a.N = up ? 4 * Co : Co; a.K = up ? Ci : 9 * Ci; a.Cg = Co;
  a.G = G; a.cpg = Co / G; a.tiles = (int)cdiv(H * W, BM); a.ntiles = (int)cdiv(a.N, BN);
  if (B * a.tiles > INT32_MAX) return fail(DVA_EUNSUPPORTED, "unet_fwd: too many pixels");
  cudaStream_t st = (cudaStream_t)stream;
  const int r2 = up ? launch_gemm<kUp2>(a, B, st, "unet_fwd") : launch_gemm<kFwdT3>(a, B, st, "unet_fwd");
  if (r2 != DVA_OK) return r2;
  const int64_t n_group = (up ? 4 : 1) * H * W * (Co / G);
  convt_stats_kernel<<<(unsigned)(B * G), kRedThreads, 0, st>>>(a.part, a.tiles, a.ntiles, G, n_group, eps, mean,
                                                                invstd);
  return check_launch("unet_fwd_stats");
}

extern "C" int dva_unet_dgrad(const float* dz, int64_t B, int64_t H, int64_t W, int Ci, int Co, const float* wd,
                              int kind, const float* add, float* dx, void* stream) {
  const int rc = check_shape("unet_dgrad", B, H, W, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (!dz || !wd || !dx) return fail(DVA_EINVAL, "unet_dgrad: null pointer");
  const bool up = kind == DVA_UNET_UP_2X2;
  ConvTArgs a{};
  a.src = dz; a.wt = wd; a.add = add; a.out = dx; a.Cs = Co;
  a.H = up ? 2 * H : H; a.W = up ? 2 * W : W; a.Ho = H; a.Wo = W;
  a.N = Ci; a.K = (up ? 4 : 9) * Co;
  a.tiles = (int)cdiv(H * W, BM);
  if (B * a.tiles > INT32_MAX) return fail(DVA_EUNSUPPORTED, "unet_dgrad: too many pixels");
  cudaStream_t st = (cudaStream_t)stream;
  return up ? launch_gemm<kDgradUp2>(a, B, st, "unet_dgrad") : launch_gemm<kDgradT3>(a, B, st, "unet_dgrad");
}

extern "C" size_t dva_unet_wgrad_workspace_bytes(int64_t B, int64_t H, int64_t W, int Ci, int Co, int kind) {
  if (B < 1 || H < 1 || W < 1 || Ci < 1 || Co < 1 || (kind != DVA_UNET_UP_2X2 && kind != DVA_UNET_T_3X3)) return 0;
  const WgradPlan p = wgrad_plan(B, H, W, Ci, Co, kind);
  return (size_t)p.splits * p.Rw * (p.Kd + 1) * sizeof(float);
}

extern "C" int dva_unet_wgrad(const float* dz, const float* x, int64_t B, int64_t H, int64_t W, int Ci, int Co,
                              int kind, float* dwf, float* dbias, void* ws, size_t ws_bytes, void* stream) {
  const int rc = check_shape("unet_wgrad", B, H, W, Ci, Co, kind);
  if (rc != DVA_OK) return rc;
  if (!dz || !x || !dwf || !dbias || !ws) return fail(DVA_EINVAL, "unet_wgrad: null pointer");
  if (ws_bytes < dva_unet_wgrad_workspace_bytes(B, H, W, Ci, Co, kind))
    return fail(DVA_EINVAL, "unet_wgrad: workspace too small");
  const WgradPlan pl = wgrad_plan(B, H, W, Ci, Co, kind);
  ConvTWgradArgs a{};
  a.dz = dz; a.x = x; a.part = (float*)ws;
  a.H = H; a.W = W; a.M = pl.M; a.rows_per_split = pl.rows_per_split;
  a.Ci = Ci; a.Co = Co; a.Rw = pl.Rw; a.Kd = pl.Kd;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)cdiv(pl.Rw, BM), (unsigned)cdiv(pl.Kd + 1, BN), (unsigned)pl.splits);
  if (kind == DVA_UNET_UP_2X2) convt_wgrad_kernel<DVA_UNET_UP_2X2><<<grid, kThreads, 0, st>>>(a);
  else convt_wgrad_kernel<DVA_UNET_T_3X3><<<grid, kThreads, 0, st>>>(a);
  const int r2 = check_launch("unet_wgrad");
  if (r2 != DVA_OK) return r2;
  convt_wgrad_reduce_kernel<<<elementwise_grid((int64_t)pl.Rw * pl.Kd + Co), kRedThreads, 0, st>>>(
      a.part, pl.splits, pl.Rw, pl.Kd, Co, dwf, dbias);
  return check_launch("unet_wgrad_reduce");
}

extern "C" int dva_unet_act(const float* z, int64_t n, float scale, float* y, void* stream) {
  if (n < 1 || !(scale > 0.f)) return fail(DVA_EINVAL, "unet_act: bad sizes or scale");
  if (!z || !y) return fail(DVA_EINVAL, "unet_act: null pointer");
  unary_act_kernel<<<elementwise_grid(n), kRedThreads, 0, (cudaStream_t)stream>>>(z, n, scale, y);
  return check_launch("unet_act");
}

extern "C" int dva_unet_act_bwd(const float* dy, const float* z, int64_t n, float scale, float* dz, void* stream) {
  if (n < 1 || !(scale > 0.f)) return fail(DVA_EINVAL, "unet_act_bwd: bad sizes or scale");
  if (!dy || !z || !dz) return fail(DVA_EINVAL, "unet_act_bwd: null pointer");
  unary_act_bwd_kernel<<<elementwise_grid(n), kRedThreads, 0, (cudaStream_t)stream>>>(dy, z, n, scale, dz);
  return check_launch("unet_act_bwd");
}
