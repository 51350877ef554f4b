// Fused feature-map pixel gather + atomic (pixel -> view) pool.
//   reference: x = self.x[(img_id per pixel, ..., py, px)]  (image.py:1285, 1871-1885) makes a
//   [P,C] copy out of the NCHW map, then BimodalCSRPool reduces it over the atomic CSR
//   (modules.py:497-500 -> pooling.py:63).  Here the [P,C] intermediate never exists: one thread
//   owns one (view, channel) output, walks the view's pixels and reads the map directly.
// With a channels-last map ([B,H,W,C]) the C channels of a pixel are one contiguous run, so a
// warp reads 32 consecutive channels per pixel (coalesced); with the reference's NCHW layout
// every element is H*W apart (32-byte sector per 4-byte element) -- supported for drop-in use,
// channels-last is the fast path.
//
// INTERP: the `interpolate=True` branch of get_mapped_features (image.py:1278-1283 ->
// sparse_interpolation, image.py:105-170): pixels live at the mapping resolution (map_w, map_h),
// the feature map is smaller, and every pixel reads 4 bilinear corners of the replicate-padded
// map.  The fp32 arithmetic follows the reference operation by operation (no FMA contraction),
// so corner choices, values and therefore max / argmax decisions are identical in fp32.
#include "bucket_sort.cuh"

namespace dva {

// Bilinear footprint of one mapping pixel (image.py:145-163).
struct Bilin {
  int r0, r1, c0, c1;          // clamped source rows / columns (replicate padding, image.py:133)
  float w00, w01, w10, w11;    // tl, tr, bl, br
};
__device__ __forceinline__ Bilin bilin_setup(int px, int py, int H, int W, float mw1, float mh1) {
  // coords = pixels / (resolution - 1), (x,y) -> (row, col)       image.py:1280-1281
  const float cy = __fdiv_rn((float)py, mh1), cx = __fdiv_rn((float)px, mw1);
  // pixels = coords * (h, w) + 0.5 in the padded frame               image.py:143
  const float p0 = __fadd_rn(__fmul_rn(cy, (float)H), 0.5f);
  const float p1 = __fadd_rn(__fmul_rn(cx, (float)W), 0.5f);
  const float top = floorf(p0), bottom = floorf(__fadd_rn(p0, 1.f));
  const float left = floorf(p1), right = floorf(__fadd_rn(p1, 1.f));
  const float dyt = __fsub_rn(p0, bottom), dyb = __fsub_rn(p0, top);   // weight of top / bottom row
  const float dxl = __fsub_rn(p1, right), dxr = __fsub_rn(p1, left);
  Bilin b;
  b.w00 = fabsf(__fmul_rn(dyt, dxl)); b.w01 = fabsf(__fmul_rn(dyt, dxr));
  b.w10 = fabsf(__fmul_rn(dyb, dxl)); b.w11 = fabsf(__fmul_rn(dyb, dxr));
  b.r0 = min(max((int)top - 1, 0), H - 1); b.r1 = min(max((int)bottom - 1, 0), H - 1);
  b.c0 = min(max((int)left - 1, 0), W - 1); b.c1 = min(max((int)right - 1, 0), W - 1);
  return b;
}

template <bool CL>
__device__ __forceinline__ int64_t fmap_off(int64_t b, int64_t c, int64_t y, int64_t x, int64_t C,
                                            int64_t H, int64_t W) {
  return CL ? (((b * H + y) * W + x) * C + c) : (((b * C + c) * H + y) * W + x);
}

// Memory safety (the reference's x[feature_map_indexing] raises IndexError on a stale or mis-scaled
// mapping; a kernel cannot raise): pixel coordinates and image ids are clamped into the map, so a bad
// mapping can never read or -- in backward -- atomically write outside the feature-map tensor.
// ops.gather_pool(check_indices=True) / DVA_CHECK_INDICES=1 validates them up front and raises.
__device__ __forceinline__ int clamp_px(int v, int n) { return v < 0 ? 0 : (v >= n ? n - 1 : v); }
__device__ __forceinline__ int64_t clamp_img(int64_t b, int64_t B) { return b < 0 ? 0 : (b >= B ? B - 1 : b); }

template <typename T, typename PIX, bool CL, int RED, bool INTERP>
__global__ void __launch_bounds__(256)
gather_pool_fwd_kernel(const T* __restrict__ fmap, const int64_t* __restrict__ img,
                       const PIX* __restrict__ pix, const int64_t* __restrict__ aptr,
                       T* __restrict__ out, int64_t* __restrict__ arg, int64_t C, int64_t H,
                       int64_t W, int64_t Vw, int64_t P, float mw1, float mh1, int64_t B) {
  const int64_t total = Vw * C;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t w = t / C, c = t - w * C;
    const int64_t p0 = aptr[w], p1 = aptr[w + 1];
    const int64_t b = clamp_img(img[w], B);
    float acc = 0.f;
    int64_t best = P;
    for (int64_t p = p0; p < p1; ++p) {
      int64_t px = (int64_t)pix[2 * p], py = (int64_t)pix[2 * p + 1];
      if (!INTERP) { px = clamp_px((int)px, (int)W); py = clamp_px((int)py, (int)H); }
      float v;
      if (INTERP) {
        const Bilin q = bilin_setup((int)px, (int)py, (int)H, (int)W, mw1, mh1);
        const float f00 = Cvt<T>::to_f(fmap[fmap_off<CL>(b, c, q.r0, q.c0, C, H, W)]);
        const float f01 = Cvt<T>::to_f(fmap[fmap_off<CL>(b, c, q.r0, q.c1, C, H, W)]);
        const float f10 = Cvt<T>::to_f(fmap[fmap_off<CL>(b, c, q.r1, q.c0, C, H, W)]);
        const float f11 = Cvt<T>::to_f(fmap[fmap_off<CL>(b, c, q.r1, q.c1, C, H, W)]);
        // image.py:165-168: four products summed left to right
        v = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q.w00, f00), __fmul_rn(q.w01, f01)),
                                __fmul_rn(q.w10, f10)), __fmul_rn(q.w11, f11));
      } else {
        v = Cvt<T>::to_f(fmap[fmap_off<CL>(b, c, py, px, C, H, W)]);
      }
      if (RED == DVA_SUM || RED == DVA_MEAN) acc += v;
      else if (p == p0 || (RED == DVA_MAX ? v > acc : v < acc)) { acc = v; best = p; }
    }
    if (RED == DVA_MEAN) acc /= (float)((p1 - p0) > 0 ? (p1 - p0) : 1);
    out[t] = Cvt<T>::from_f(acc);
    // the arg table is only needed (and only written) for views with two or more pixels; a
    // one-pixel view (every view under exact splatting) routes its gradient to that pixel
    if ((RED == DVA_MAX || RED == DVA_MIN) && arg != nullptr && p1 - p0 >= 2) arg[t] = best;
  }
}

template <bool CL, bool INTERP, typename PIX>
__device__ __forceinline__ void scatter_pixel(float* __restrict__ gfmap, const PIX* __restrict__ pix,
                                              int64_t p, int64_t b, int64_t c, int64_t C, int64_t H,
                                              int64_t W, float mw1, float mh1, float g) {
  int64_t px = (int64_t)pix[2 * p], py = (int64_t)pix[2 * p + 1];
  if (!INTERP) { px = clamp_px((int)px, (int)W); py = clamp_px((int)py, (int)H); }
  if (INTERP) {
    const Bilin q = bilin_setup((int)px, (int)py, (int)H, (int)W, mw1, mh1);
    atomicAdd(gfmap + fmap_off<CL>(b, c, q.r0, q.c0, C, H, W), q.w00 * g);
    atomicAdd(gfmap + fmap_off<CL>(b, c, q.r0, q.c1, C, H, W), q.w01 * g);
    atomicAdd(gfmap + fmap_off<CL>(b, c, q.r1, q.c0, C, H, W), q.w10 * g);
    atomicAdd(gfmap + fmap_off<CL>(b, c, q.r1, q.c1, C, H, W), q.w11 * g);
  } else {
    atomicAdd(gfmap + fmap_off<CL>(b, c, py, px, C, H, W), g);
  }
}

template <typename T, typename PIX, bool CL, int RED, bool INTERP>
__global__ void __launch_bounds__(256)
gather_pool_bwd_kernel(const T* __restrict__ gout, const int64_t* __restrict__ img,
                       const PIX* __restrict__ pix, const int64_t* __restrict__ aptr,
                       const int64_t* __restrict__ arg, float* __restrict__ gfmap, int64_t C,
                       int64_t H, int64_t W, int64_t Vw, float mw1, float mh1, int64_t B) {
  const int64_t total = Vw * C;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t w = t / C, c = t - w * C;
    const int64_t p0 = aptr[w], p1 = aptr[w + 1];
    if (p1 <= p0) continue;
    const int64_t b = clamp_img(img[w], B);
    float g = Cvt<T>::to_f(gout[t]);
    if (RED == DVA_MEAN) g /= (float)(p1 - p0);
    if (RED == DVA_MAX || RED == DVA_MIN) {
      scatter_pixel<CL, INTERP>(gfmap, pix, (p1 - p0 == 1) ? p0 : arg[t], b, c, C, H, W, mw1, mh1, g);
    } else {
      for (int64_t p = p0; p < p1; ++p) scatter_pixel<CL, INTERP>(gfmap, pix, p, b, c, C, H, W, mw1, mh1, g);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// channels-last vector path: LPR lanes own the 16-byte chunks of one view's output row, a warp
// works on 32/LPR views per step and kGpUnroll steps at once (their index loads, pixel loads and
// row-chunk loads are issued back to back), so a pixel costs one LDG.128 per lane instead of
// VEC scalar loads plus 64-bit index arithmetic per channel.  Same arithmetic as the scalar kernel
// (the bilinear branch keeps the reference's fp32 operation order).
// ---------------------------------------------------------------------------------------------
constexpr int kGpWarps = 8;

template <typename T, typename PIX, bool INTERP> struct PixLoad {
  static constexpr int VEC = Vec16<T>::N;
  uint4 raw[INTERP ? 4 : 1];
  Bilin q;
  // fb: map of the view's image + this lane's chunk offset (bytes); pixel_bytes = C * sizeof(T)
  __device__ __forceinline__ void issue(const char* __restrict__ fb, const PIX* __restrict__ pix, int64_t p,
                                        int H, int W, uint32_t pixel_bytes, float mw1, float mh1) {
    int px = (int)pix[2 * p], py = (int)pix[2 * p + 1];
    if constexpr (!INTERP) { px = clamp_px(px, W); py = clamp_px(py, H); }
    if constexpr (INTERP) {
      q = bilin_setup(px, py, H, W, mw1, mh1);
      raw[0] = ldg_stream16(fb + ((int64_t)q.r0 * W + q.c0) * pixel_bytes);
      raw[1] = ldg_stream16(fb + ((int64_t)q.r0 * W + q.c1) * pixel_bytes);
      raw[2] = ldg_stream16(fb + ((int64_t)q.r1 * W + q.c0) * pixel_bytes);
      raw[3] = ldg_stream16(fb + ((int64_t)q.r1 * W + q.c1) * pixel_bytes);
    } else {
      raw[0] = ldg_stream16(fb + ((int64_t)py * W + px) * pixel_bytes);
    }
  }
  __device__ __forceinline__ void value(float (&v)[VEC]) const {
    if constexpr (INTERP) {
      float f00[VEC], f01[VEC], f10[VEC], f11[VEC];
      unpack16<T, VEC>(raw[0], f00); unpack16<T, VEC>(raw[1], f01);
      unpack16<T, VEC>(raw[2], f10); unpack16<T, VEC>(raw[3], f11);
#pragma unroll
      for (int j = 0; j < VEC; ++j)   // image.py:165-168: four products summed left to right
        v[j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q.w00, f00[j]), __fmul_rn(q.w01, f01[j])),
                                   __fmul_rn(q.w10, f10[j])), __fmul_rn(q.w11, f11[j]));
    } else {
      unpack16<T, VEC>(raw[0], v);
    }
  }
};

template <typename T, typename PIX, int LPR, int RED, bool INTERP>
__global__ void __launch_bounds__(kGpWarps * 32)
gather_pool_fwd_cl_kernel(const T* __restrict__ fmap, const int64_t* __restrict__ img,
                          const PIX* __restrict__ pix, const int64_t* __restrict__ aptr,
                          T* __restrict__ out, int64_t* __restrict__ arg, int C, int H, int W,
                          int64_t Vw, int64_t P, float mw1, float mh1, int64_t B) {
  constexpr int VEC = Vec16<T>::N, RPI = 32 / LPR, U = INTERP ? 2 : 4;
  const int lane = threadIdx.x & 31, sg = lane / LPR, lir = lane % LPR;
  const int cv = C / VEC, tiles = (cv + LPR - 1) / LPR;
  const int64_t items = Vw * tiles;
  const uint32_t pixel_bytes = (uint32_t)C * sizeof(T);
  const int64_t map_bytes = (int64_t)H * W * pixel_bytes;
  const char* __restrict__ fbase = reinterpret_cast<const char*>(fmap);
  const int64_t gwarp = (int64_t)blockIdx.x * kGpWarps + (threadIdx.x >> 5);
  const int64_t stride = (int64_t)gridDim.x * kGpWarps * RPI * U;
  for (int64_t it0 = gwarp * RPI * U; it0 < items; it0 += stride) {
    int64_t w[U], p0[U]; int n[U], ck[U]; bool act[U];
    const char* fb[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t item = it0 + u * RPI + sg;
      act[u] = item < items;
      w[u] = act[u] ? (tiles == 1 ? item : item / tiles) : 0;
      ck[u] = (int)(item - w[u] * tiles) * LPR + lir;
      act[u] = act[u] && ck[u] < cv;
      p0[u] = aptr[w[u]];
      n[u] = (int)(aptr[w[u] + 1] - p0[u]);
      fb[u] = fbase + clamp_img(img[w[u]], B) * map_bytes + (act[u] ? ck[u] * 16 : 0);
    }
    PixLoad<T, PIX, INTERP> pl[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (n[u] > 0) pl[u].issue(fb[u], pix, p0[u], H, W, pixel_bytes, mw1, mh1);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float acc[VEC]; int best[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) { acc[j] = 0.f; best[j] = 0; }
      if (n[u] > 0) pl[u].value(acc);
      for (int k = 1; k < n[u]; ++k) {              // two or more pixels per view: not under exact splatting
        PixLoad<T, PIX, INTERP> nx;
        nx.issue(fb[u], pix, p0[u] + k, H, W, pixel_bytes, mw1, mh1);
        float v[VEC];
        nx.value(v);
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          if (RED == DVA_SUM || RED == DVA_MEAN) acc[j] += v[j];
          else if (RED == DVA_MAX ? v[j] > acc[j] : v[j] < acc[j]) { acc[j] = v[j]; best[j] = k; }
        }
      }
      if (RED == DVA_MEAN && n[u] > 1) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] /= (float)n[u];
      }
      if (act[u]) {
        const int64_t e0 = w[u] * C + (int64_t)ck[u] * VEC;
        stg_stream16(reinterpret_cast<char*>(out) + e0 * sizeof(T), pack16<T, VEC>(acc));
        if ((RED == DVA_MAX || RED == DVA_MIN) && arg != nullptr && n[u] >= 2) {
#pragma unroll
          for (int j = 0; j < VEC; ++j) arg[e0 + j] = p0[u] + best[j];
        }
      }
    }
  }
}

template <typename PIX, bool INTERP, int VEC>
__device__ __forceinline__ void scatter_chunk(float* __restrict__ gmap_b /* image + chunk offset */,
                                              const PIX* __restrict__ pix, int64_t p, int C, int H, int W,
                                              float mw1, float mh1, const float (&g)[VEC]) {
  int px = (int)pix[2 * p], py = (int)pix[2 * p + 1];
  if constexpr (!INTERP) { px = clamp_px(px, W); py = clamp_px(py, H); }
  if constexpr (INTERP) {
    const Bilin q = bilin_setup(px, py, H, W, mw1, mh1);
    const int64_t o[4] = {((int64_t)q.r0 * W + q.c0) * C, ((int64_t)q.r0 * W + q.c1) * C,
                          ((int64_t)q.r1 * W + q.c0) * C, ((int64_t)q.r1 * W + q.c1) * C};
    const float wq[4] = {q.w00, q.w01, q.w10, q.w11};
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int j = 0; j < VEC; j += 4)
        red_add_v4(gmap_b + o[k] + j, wq[k] * g[j], wq[k] * g[j + 1], wq[k] * g[j + 2], wq[k] * g[j + 3]);
  } else {
    float* a = gmap_b + ((int64_t)py * W + px) * C;
#pragma unroll
    for (int j = 0; j < VEC; j += 4) red_add_v4(a + j, g[j], g[j + 1], g[j + 2], g[j + 3]);
  }
}

template <typename T, typename PIX, int LPR, int RED, bool INTERP>
__global__ void __launch_bounds__(kGpWarps * 32)
gather_pool_bwd_cl_kernel(const T* __restrict__ gout, const int64_t* __restrict__ img,
                          const PIX* __restrict__ pix, const int64_t* __restrict__ aptr,
                          const int64_t* __restrict__ arg, float* __restrict__ gfmap, int C, int H,
                          int W, int64_t Vw, float mw1, float mh1, int64_t B) {
  constexpr int VEC = Vec16<T>::N, RPI = 32 / LPR, U = 4;
  const int lane = threadIdx.x & 31, sg = lane / LPR, lir = lane % LPR;
  const int cv = C / VEC, tiles = (cv + LPR - 1) / LPR;
  const int64_t items = Vw * tiles;
  const int64_t map_elems = (int64_t)H * W * C;
  const int64_t gwarp = (int64_t)blockIdx.x * kGpWarps + (threadIdx.x >> 5);
  const int64_t stride = (int64_t)gridDim.x * kGpWarps * RPI * U;
  for (int64_t it0 = gwarp * RPI * U; it0 < items; it0 += stride) {
    int64_t w[U], p0[U], b[U]; int n[U], ck[U]; bool act[U];
    uint4 raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t item = it0 + u * RPI + sg;
      act[u] = item < items;
      w[u] = act[u] ? (tiles == 1 ? item : item / tiles) : 0;
      ck[u] = (int)(item - w[u] * tiles) * LPR + lir;
      act[u] = act[u] && ck[u] < cv;
      p0[u] = aptr[w[u]];
      n[u] = (int)(aptr[w[u] + 1] - p0[u]);
      b[u] = clamp_img(img[w[u]], B);
      act[u] = act[u] && n[u] > 0;
      if (act[u]) raw[u] = ldg_stream16(reinterpret_cast<const char*>(gout) + (w[u] * C + (int64_t)ck[u] * VEC) * sizeof(T));
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!act[u]) continue;
      float g[VEC];
      unpack16<T, VEC>(raw[u], g);
      if (RED == DVA_MEAN) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) g[j] /= (float)n[u];
      }
      const int c0 = ck[u] * VEC;
      float* gm = gfmap + b[u] * map_elems + c0;
      if (RED == DVA_MAX || RED == DVA_MIN) {
        if (n[u] == 1) {
          scatter_chunk<PIX, INTERP, VEC>(gm, pix, p0[u], C, H, W, mw1, mh1, g);
        } else {                                    // per-channel winners: scalar atomics
          const int64_t e0 = w[u] * C + c0;
#pragma unroll
          for (int j = 0; j < VEC; ++j)
            scatter_pixel<true, INTERP>(gfmap, pix, arg[e0 + j], b[u], c0 + j, C, H, W, mw1, mh1, g[j]);
        }
      } else {
        for (int k = 0; k < n[u]; ++k) scatter_chunk<PIX, INTERP, VEC>(gm, pix, p0[u] + k, C, H, W, mw1, mh1, g);
      }
    }
  }
}

template <typename T> static bool gp_cl_vec_ok(const void* map, const void* rows, int64_t C, int64_t H, int64_t W) {
  return vec16_ok<T>(C, map, rows) && C < (1 << 20) && H * W < (1ll << 31);
}

// f(T{}, PIX{}, std::bool_constant<CL>{}, std::integral_constant<int, RED>{}) for the storage type, pixel
// coordinate type (int16 / int32), map layout (channels-last / NCHW) and reduce of a call
template <typename F>
static int gp_dispatch(const char* who, int dtype, int reduce, int channels_last, int pix_is_i16, F&& f) {
  if (!known_dtype(dtype)) return failf(DVA_EINVAL, "%s: unknown dtype", who);
  int rc = DVA_OK;
  const bool known = with_reduce(reduce, [&](auto red) {
    rc = with_dtype(dtype, [&](auto t) {
      auto pix = [&](auto cl) { return pix_is_i16 ? f(t, int16_t{}, cl, red) : f(t, int32_t{}, cl, red); };
      return channels_last ? pix(std::true_type{}) : pix(std::false_type{});
    });
  });
  return known ? rc : failf(DVA_EINVAL, "%s: unknown reduce", who);
}

template <typename T, typename PIX, bool CL, int RED, bool INTERP>
static int gp_fwd(const void* fmap, const int64_t* img, const void* pix, const int64_t* aptr,
                  void* out, int64_t* arg, int64_t C, int64_t H, int64_t W, int64_t Vw,
                  int64_t P, float mw1, float mh1, cudaStream_t st, int64_t B) {
  if constexpr (CL) {
    if (gp_cl_vec_ok<T>(fmap, out, C, H, W)) {
      const int64_t cv = C / Vec16<T>::N;
      with_lpr(cv, [&](auto lpr) {
        constexpr int LPR = decltype(lpr)::value;
        const int grid = grid_cap(Vw * ((cv + LPR - 1) / LPR), kGpWarps * (32 / LPR) * (INTERP ? 2 : 4), 8);
        gather_pool_fwd_cl_kernel<T, PIX, LPR, RED, INTERP><<<grid, kGpWarps * 32, 0, st>>>(
            (const T*)fmap, img, (const PIX*)pix, aptr, (T*)out, arg, (int)C, (int)H, (int)W, Vw, P, mw1, mh1, B);
      });
      return check_launch("gather_pool_fwd(cl)");
    }
  }
  gather_pool_fwd_kernel<T, PIX, CL, RED, INTERP><<<grid_cap(Vw * C, 256, 16), 256, 0, st>>>(
      (const T*)fmap, img, (const PIX*)pix, aptr, (T*)out, arg, C, H, W, Vw, P, mw1, mh1, B);
  return check_launch("gather_pool_fwd");
}

template <typename T, typename PIX, bool CL, int RED, bool INTERP>
static int gp_bwd(const void* gout, const int64_t* img, const void* pix, const int64_t* aptr,
                  const int64_t* arg, float* gfmap, int64_t C, int64_t H, int64_t W,
                  int64_t Vw, float mw1, float mh1, cudaStream_t st, int64_t B) {
  if constexpr (CL) {
    if (gp_cl_vec_ok<T>(gfmap, gout, C, H, W) && C % 4 == 0) {
      const int64_t cv = C / Vec16<T>::N;
      with_lpr(cv, [&](auto lpr) {
        constexpr int LPR = decltype(lpr)::value;
        const int grid = grid_cap(Vw * ((cv + LPR - 1) / LPR), kGpWarps * (32 / LPR) * 4, 8);
        gather_pool_bwd_cl_kernel<T, PIX, LPR, RED, INTERP><<<grid, kGpWarps * 32, 0, st>>>(
            (const T*)gout, img, (const PIX*)pix, aptr, arg, gfmap, (int)C, (int)H, (int)W, Vw, mw1, mh1, B);
      });
      return check_launch("gather_pool_bwd(cl)");
    }
  }
  gather_pool_bwd_kernel<T, PIX, CL, RED, INTERP><<<grid_cap(Vw * C, 256, 16), 256, 0, st>>>(
      (const T*)gout, img, (const PIX*)pix, aptr, arg, gfmap, C, H, W, Vw, mw1, mh1, B);
  return check_launch("gather_pool_bwd");
}

}  // namespace dva

using namespace dva;

template <bool INTERP>
static int gather_pool_fwd_impl(const char* who, const void* fmap, int channels_last, const int64_t* img,
                                const void* pix, int pix_is_i16, const int64_t* aptr, void* out,
                                int64_t* arg, int64_t B, int64_t C, int64_t H, int64_t W,
                                int64_t map_w, int64_t map_h, int64_t Vw, int64_t P, int reduce,
                                int dtype, void* stream) {
  if (B < 0 || C < 0 || H < 0 || W < 0 || Vw < 0 || P < 0) return failf(DVA_EINVAL, "%s: negative size", who);
  if (Vw == 0 || C == 0) return DVA_OK;
  if (P > 0 && (B < 1 || H < 1 || W < 1)) return failf(DVA_EINVAL, "%s: pixels given but the map is empty", who);
  if (!aptr || !out || !img || (P > 0 && (!fmap || !pix))) return failf(DVA_EINVAL, "%s: null pointer", who);
  if (INTERP && (map_w < 2 || map_h < 2 || H < 1 || W < 1 || H > (1 << 24) || W > (1 << 24)))
    return failf(DVA_EINVAL, "%s: bad map / mapping size", who);
  const float mw1 = (float)(map_w - 1), mh1 = (float)(map_h - 1);
  cudaStream_t st = (cudaStream_t)stream;
  return gp_dispatch(who, dtype, reduce, channels_last, pix_is_i16, [&](auto t, auto p, auto cl, auto red) {
    return gp_fwd<decltype(t), decltype(p), decltype(cl)::value, decltype(red)::value, INTERP>(
        fmap, img, pix, aptr, out, arg, C, H, W, Vw, P, mw1, mh1, st, B);
  });
}

template <bool INTERP>
static int gather_pool_bwd_impl(const char* who, const void* grad_out, int channels_last,
                                const int64_t* img, const void* pix, int pix_is_i16,
                                const int64_t* aptr, const int64_t* arg, float* grad_fmap, int64_t B,
                                int64_t C, int64_t H, int64_t W, int64_t map_w, int64_t map_h,
                                int64_t Vw, int64_t P, int reduce, int dtype, void* stream) {
  if (B < 0 || C < 0 || H < 0 || W < 0 || Vw < 0 || P < 0) return failf(DVA_EINVAL, "%s: negative size", who);
  if (Vw == 0 || C == 0 || P == 0) return DVA_OK;
  if (B < 1 || H < 1 || W < 1) return failf(DVA_EINVAL, "%s: pixels given but the map is empty", who);
  if (!aptr || !grad_out || !img || !pix || !grad_fmap) return failf(DVA_EINVAL, "%s: null pointer", who);
  if ((reduce == DVA_MAX || reduce == DVA_MIN) && !arg) return failf(DVA_EINVAL, "%s: max/min need arg", who);
  if (INTERP && (map_w < 2 || map_h < 2 || H < 1 || W < 1 || H > (1 << 24) || W > (1 << 24)))
    return failf(DVA_EINVAL, "%s: bad map / mapping size", who);
  const float mw1 = (float)(map_w - 1), mh1 = (float)(map_h - 1);
  cudaStream_t st = (cudaStream_t)stream;
  return gp_dispatch(who, dtype, reduce, channels_last, pix_is_i16, [&](auto t, auto p, auto cl, auto red) {
    return gp_bwd<decltype(t), decltype(p), decltype(cl)::value, decltype(red)::value, INTERP>(
        grad_out, img, pix, aptr, arg, grad_fmap, C, H, W, Vw, mw1, mh1, st, B);
  });
}

extern "C" int dva_gather_pool_fwd(const void* fmap, int channels_last, const int64_t* img,
                                   const void* pix, int pix_is_i16, const int64_t* aptr,
                                   void* out, int64_t* arg, int64_t B, int64_t C, int64_t H,
                                   int64_t W, int64_t Vw, int64_t P, int reduce, int dtype,
                                   void* stream) {
  return gather_pool_fwd_impl<false>("gather_pool_fwd", fmap, channels_last, img, pix, pix_is_i16, aptr,
                                     out, arg, B, C, H, W, 0, 0, Vw, P, reduce, dtype, stream);
}

extern "C" int dva_gather_pool_bwd(const void* grad_out, int channels_last, const int64_t* img,
                                   const void* pix, int pix_is_i16, const int64_t* aptr,
                                   const int64_t* arg, float* grad_fmap, int64_t B, int64_t C,
                                   int64_t H, int64_t W, int64_t Vw, int64_t P, int reduce,
                                   int dtype, void* stream) {
  return gather_pool_bwd_impl<false>("gather_pool_bwd", grad_out, channels_last, img, pix, pix_is_i16,
                                     aptr, arg, grad_fmap, B, C, H, W, 0, 0, Vw, P, reduce, dtype, stream);
}

extern "C" int dva_interp_pool_fwd(const void* fmap, int channels_last, const int64_t* img,
                                   const void* pix, int pix_is_i16, const int64_t* aptr,
                                   void* out, int64_t* arg, int64_t B, int64_t C, int64_t H,
                                   int64_t W, int64_t map_w, int64_t map_h, int64_t Vw, int64_t P,
                                   int reduce, int dtype, void* stream) {
  return gather_pool_fwd_impl<true>("interp_pool_fwd", fmap, channels_last, img, pix, pix_is_i16, aptr,
                                    out, arg, B, C, H, W, map_w, map_h, Vw, P, reduce, dtype, stream);
}

extern "C" int dva_interp_pool_bwd(const void* grad_out, int channels_last, const int64_t* img,
                                   const void* pix, int pix_is_i16, const int64_t* aptr,
                                   const int64_t* arg, float* grad_fmap, int64_t B, int64_t C,
                                   int64_t H, int64_t W, int64_t map_w, int64_t map_h, int64_t Vw,
                                   int64_t P, int reduce, int dtype, void* stream) {
  return gather_pool_bwd_impl<true>("interp_pool_bwd", grad_out, channels_last, img, pix, pix_is_i16,
                                    aptr, arg, grad_fmap, B, C, H, W, map_w, map_h, Vw, P, reduce, dtype, stream);
}

// ---------------------------------------------------------------------------------------------
// Deterministic backward (used under torch.use_deterministic_algorithms): instead of scattering
// every contribution with fp32 atomics, the contributions are bucketed by map pixel and every map
// element is summed by one owner in a fixed order.  For element (b, y, x, c):
//   contributions (p, k): pixel slot p (atomic-CSR order) of view w; k = 0 for the plain gather,
//     k = 0..3 = corners w00, w01, w10, w11 of bilin_setup for the bilinear path (two corners of one
//     slot clamped onto the same pixel are two contributions); taken in ascending (p, k);
//   value: g = float(grad_out[w, c]); mean: __fdiv_rn(g, n_w); max / min: only when n_w == 1 or
//     arg[w, c] == p; bilinear: __fmul_rn(w_k, value);
//   sum: acc = +0.0f, acc = __fadd_rn(acc, value) (explicit _rn: no FMA contraction).
// Index: counting sort of the contribution ids p * K + k by pixel key (b * H + y) * W + x
// (bucket_sort.cuh: histogram, scan, scatter, per-bucket rank sort), then one pass that stores the
// view and bilinear weight beside every ordered entry.  The reducers write every element of the map
// gradient, zeros included.  The result is a pure function of the inputs.
// ---------------------------------------------------------------------------------------------
namespace dva {
namespace det {

// view of every pixel slot (-1: in no view); one warp per view
__global__ void __launch_bounds__(256)
slot_views_kernel(const int64_t* __restrict__ aptr, int64_t Vw, int64_t P, int64_t* __restrict__ view_of) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < Vw; w += warps) {
    const int64_t p0 = max(aptr[w], (int64_t)0), p1 = min(aptr[w + 1], P);
    for (int64_t p = p0 + lane; p < p1; p += 32) view_of[p] = w;
  }
}

// bucket keys of slot p: the map pixel of each of its K contributions (clamped like the forward)
template <typename PIX, bool INTERP>
struct PixelKey {
  const int64_t* view_of; const int64_t* img; const PIX* pix; int64_t B; int H, W; float mw1, mh1;
  __device__ __forceinline__ void operator()(int64_t p, int64_t (&k)[INTERP ? 4 : 1]) const {
    const int64_t w = view_of[p];
    if (w < 0) {
#pragma unroll
      for (int j = 0; j < (INTERP ? 4 : 1); ++j) k[j] = -1;
      return;
    }
    const int64_t row0 = clamp_img(img[w], B) * H;
    const int px = (int)pix[2 * p], py = (int)pix[2 * p + 1];
    if constexpr (INTERP) {
      const Bilin q = bilin_setup(px, py, H, W, mw1, mh1);
      k[0] = (row0 + q.r0) * W + q.c0; k[1] = (row0 + q.r0) * W + q.c1;
      k[2] = (row0 + q.r1) * W + q.c0; k[3] = (row0 + q.r1) * W + q.c1;
    } else {
      k[0] = (row0 + clamp_px(py, H)) * W + clamp_px(px, W);
    }
  }
};

// what the reducers need of an ordered entry: its view and (bilinear) corner weight
struct Ent { int32_t w; float wt; };

template <typename PIX, bool INTERP>
__global__ void __launch_bounds__(256)
describe_entries(const int64_t* __restrict__ sorted, const int64_t* __restrict__ n_entries, int64_t bound,
                 const int64_t* __restrict__ view_of, const PIX* __restrict__ pix, int H, int W, float mw1,
                 float mh1, Ent* __restrict__ ent) {
  const int64_t n = min(*n_entries, bound);
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t cid = sorted[e];
    const int64_t p = INTERP ? (cid >> 2) : cid;
    Ent d;
    d.w = (int32_t)view_of[p];
    d.wt = 1.f;
    if constexpr (INTERP) {
      const Bilin q = bilin_setup((int)pix[2 * p], (int)pix[2 * p + 1], H, W, mw1, mh1);
      const int k = (int)(cid & 3);
      d.wt = k == 0 ? q.w00 : (k == 1 ? q.w01 : (k == 2 ? q.w10 : q.w11));
    }
    ent[e] = d;
  }
}

template <int RED, bool INTERP>
__device__ __forceinline__ float contrib(float g, int n, float wt) {
  if (RED == DVA_MEAN) g = __fdiv_rn(g, (float)n);
  if (INTERP) g = __fmul_rn(wt, g);
  return g;
}

// channels-last, whole 16-byte chunks: LPR lanes own the chunks of one map pixel (the sub-warp shape of
// gather_pool_bwd_cl_kernel), walk its entries in order and gather the grad_out rows of their views
template <typename T, int LPR, int RED, bool INTERP>
__global__ void __launch_bounds__(kGpWarps * 32)
gather_pool_bwd_det_cl_kernel(const T* __restrict__ gout, const int64_t* __restrict__ aptr,
                              const int64_t* __restrict__ arg, const int64_t* __restrict__ off,
                              const int64_t* __restrict__ sorted, const Ent* __restrict__ ent,
                              float* __restrict__ gfmap, int C, int64_t NB) {
  constexpr int VEC = Vec16<T>::N, RPI = 32 / LPR;
  const int lane = threadIdx.x & 31, sg = lane / LPR, lir = lane % LPR;
  const int cv = C / VEC, tiles = (cv + LPR - 1) / LPR;
  const int64_t items = NB * tiles;
  const int64_t stride = (int64_t)gridDim.x * kGpWarps * RPI;
  for (int64_t item = ((int64_t)blockIdx.x * kGpWarps + (threadIdx.x >> 5)) * RPI + sg; item < items; item += stride) {
    const int64_t q = tiles == 1 ? item : item / tiles;
    const int ck = (int)(item - q * tiles) * LPR + lir;
    if (ck >= cv) continue;
    const int64_t e1 = off[q + 1];
    float acc[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
    for (int64_t e = off[q]; e < e1; ++e) {
      const Ent d = ent[e];
      const int64_t w = d.w;
      const int n = RED == DVA_SUM ? 1 : (int)(aptr[w + 1] - aptr[w]);
      float g[VEC];
      unpack16<T, VEC>(__ldg(reinterpret_cast<const uint4*>(gout + w * C + (int64_t)ck * VEC)), g);
      bool on[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) on[j] = true;
      if ((RED == DVA_MAX || RED == DVA_MIN) && n >= 2) {
        const int64_t p = INTERP ? (sorted[e] >> 2) : sorted[e];
        const int64_t* a = arg + w * C + (int64_t)ck * VEC;
#pragma unroll
        for (int j = 0; j < VEC; ++j) on[j] = a[j] == p;
      }
#pragma unroll
      for (int j = 0; j < VEC; ++j)
        if (on[j]) acc[j] = __fadd_rn(acc[j], contrib<RED, INTERP>(g[j], n, d.wt));
    }
    float4* o = reinterpret_cast<float4*>(gfmap + q * C + (int64_t)ck * VEC);
#pragma unroll
    for (int j = 0; j < VEC; j += 4) o[j / 4] = make_float4(acc[j], acc[j + 1], acc[j + 2], acc[j + 3]);
  }
}

// one thread per map-gradient element: NCHW maps and channels-last rows that are not whole 16-byte chunks
template <typename T, bool CL, int RED, bool INTERP>
__global__ void __launch_bounds__(256)
gather_pool_bwd_det_kernel(const T* __restrict__ gout, const int64_t* __restrict__ aptr,
                           const int64_t* __restrict__ arg, const int64_t* __restrict__ off,
                           const int64_t* __restrict__ sorted, const Ent* __restrict__ ent,
                           float* __restrict__ gfmap, int64_t C, int64_t HW, int64_t total) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t q, c;
    if (CL) {
      q = t / C; c = t - q * C;
    } else {                                      // t = (b * C + c) * HW + s  ->  q = b * HW + s
      const int64_t bc = t / HW, s = t - bc * HW, b = bc / C;
      c = bc - b * C; q = b * HW + s;
    }
    const int64_t e1 = off[q + 1];
    float acc = 0.f;
    for (int64_t e = off[q]; e < e1; ++e) {
      const Ent d = ent[e];
      const int64_t w = d.w;
      const int n = RED == DVA_SUM ? 1 : (int)(aptr[w + 1] - aptr[w]);
      if ((RED == DVA_MAX || RED == DVA_MIN) && n >= 2 && arg[w * C + c] != (INTERP ? (sorted[e] >> 2) : sorted[e]))
        continue;
      acc = __fadd_rn(acc, contrib<RED, INTERP>(Cvt<T>::to_f(gout[w * C + c]), n, d.wt));
    }
    gfmap[t] = acc;
  }
}

struct Workspace {
  int64_t* view_of;
  Ent* ent;
  bk::BucketIndex idx;
};

static size_t carve(uint8_t* base, int64_t P, int64_t n_entries, int64_t NB, Workspace* w) {
  size_t o = 0;
  auto take = [&](size_t bytes) { uint8_t* p = base ? base + o : nullptr; o += round256(bytes); return p; };
  uint8_t* p;
  p = take((size_t)(P + 1) * 8); if (w) w->view_of = (int64_t*)p;
  p = take((size_t)(n_entries + 1) * sizeof(Ent)); if (w) w->ent = (Ent*)p;
  o += bk::carve_index(base ? base + o : nullptr, n_entries, NB, w ? &w->idx : nullptr);
  return o;
}

static size_t workspace_bytes(int64_t B, int64_t H, int64_t W, int64_t P, int K) {
  if (B < 0 || H < 0 || W < 0 || P < 0) return 0;
  return carve(nullptr, P, P * K, B * H * W, nullptr) + 256;
}

template <typename T, typename PIX, bool CL, int RED, bool INTERP>
static int gp_bwd_det(const void* gout, const int64_t* img, const void* pix, const int64_t* aptr,
                      const int64_t* arg, float* gfmap, int64_t B, int64_t C, int64_t H, int64_t W,
                      int64_t Vw, int64_t P, float mw1, float mh1, void* workspace, cudaStream_t st) {
  constexpr int K = INTERP ? 4 : 1;
  const int64_t NB = B * H * W;
  Workspace ws;
  carve(align256(workspace), P, P * K, NB, &ws);
  cudaError_t e = cudaMemsetAsync(ws.view_of, 0xff, (size_t)P * 8, st);           // -1: slot in no view
  if (e != cudaSuccess) return fail((int)e, "gather_pool_bwd_det: memset failed");
  slot_views_kernel<<<grid_cap(Vw * 32, 256, 16), 256, 0, st>>>(aptr, Vw, P, ws.view_of);
  int rc = check_launch("gp_det_slot_views");
  if (rc) return rc;
  const PixelKey<PIX, INTERP> key{ws.view_of, img, (const PIX*)pix, B, (int)H, (int)W, mw1, mh1};
  if ((rc = bk::build_index<K>(key, P, NB, ws.idx, st))) return rc;
  describe_entries<PIX, INTERP><<<grid_cap(P * K, 256, 16), 256, 0, st>>>(ws.idx.sorted, ws.idx.off + NB, P * K, ws.view_of,
                                                                           (const PIX*)pix, (int)H, (int)W, mw1, mh1, ws.ent);
  if ((rc = check_launch("gp_det_describe_entries"))) return rc;
  const T* g = (const T*)gout;
  if constexpr (CL) {
    if (gp_cl_vec_ok<T>(gfmap, gout, C, H, W) && C % 4 == 0) {
      const int64_t cv = C / Vec16<T>::N;
      with_lpr(cv, [&](auto lpr) {
        constexpr int LPR = decltype(lpr)::value;
        const int grid = grid_cap(NB * ((cv + LPR - 1) / LPR), kGpWarps * (32 / LPR), 8);
        gather_pool_bwd_det_cl_kernel<T, LPR, RED, INTERP><<<grid, kGpWarps * 32, 0, st>>>(
            g, aptr, arg, ws.idx.off, ws.idx.sorted, ws.ent, gfmap, (int)C, NB);
      });
      return check_launch("gather_pool_bwd_det(cl)");
    }
  }
  const int64_t total = NB * C;
  gather_pool_bwd_det_kernel<T, CL, RED, INTERP><<<grid_cap(total, 256, 16), 256, 0, st>>>(
      g, aptr, arg, ws.idx.off, ws.idx.sorted, ws.ent, gfmap, C, H * W, total);
  return check_launch("gather_pool_bwd_det");
}

}  // namespace det
}  // namespace dva

template <bool INTERP>
static int gather_pool_bwd_det_impl(const char* who, const void* grad_out, int channels_last,
                                    const int64_t* img, const void* pix, int pix_is_i16,
                                    const int64_t* aptr, const int64_t* arg, float* grad_fmap, int64_t B,
                                    int64_t C, int64_t H, int64_t W, int64_t map_w, int64_t map_h,
                                    int64_t Vw, int64_t P, int reduce, int dtype, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  if (B < 0 || C < 0 || H < 0 || W < 0 || Vw < 0 || P < 0) return failf(DVA_EINVAL, "%s: negative size", who);
  if (reduce < DVA_SUM || reduce > DVA_MIN) return failf(DVA_EINVAL, "%s: unknown reduce", who);
  if (!known_dtype(dtype)) return failf(DVA_EINVAL, "%s: unknown dtype", who);
  const bool work = Vw > 0 && P > 0;
  if (work && C > 0 && (B < 1 || H < 1 || W < 1)) return failf(DVA_EINVAL, "%s: pixels given but the map is empty", who);
  if (B * C * H * W == 0) return DVA_OK;
  if (!grad_fmap) return failf(DVA_EINVAL, "%s: null pointer", who);
  cudaStream_t st = (cudaStream_t)stream;
  if (!work) {          // no contribution: the map gradient is all zeros
    cudaError_t e = cudaMemsetAsync(grad_fmap, 0, (size_t)(B * C * H * W) * 4, st);
    return e == cudaSuccess ? DVA_OK : failf((int)e, "%s: memset failed", who);
  }
  if (!aptr || !grad_out || !img || !pix || !workspace) return failf(DVA_EINVAL, "%s: null pointer", who);
  if ((reduce == DVA_MAX || reduce == DVA_MIN) && !arg) return failf(DVA_EINVAL, "%s: max/min need arg", who);
  if (INTERP && (map_w < 2 || map_h < 2 || H > (1 << 24) || W > (1 << 24)))
    return failf(DVA_EINVAL, "%s: bad map / mapping size", who);
  if (Vw >= (1ll << 31)) return failf(DVA_EUNSUPPORTED, "%s: more than 2^31 views", who);
  if (workspace_bytes < det::workspace_bytes(B, H, W, P, INTERP ? 4 : 1))
    return failf(DVA_EINVAL, "%s: workspace too small", who);
  const float mw1 = (float)(map_w - 1), mh1 = (float)(map_h - 1);
  return gp_dispatch(who, dtype, reduce, channels_last, pix_is_i16, [&](auto t, auto p, auto cl, auto red) {
    return det::gp_bwd_det<decltype(t), decltype(p), decltype(cl)::value, decltype(red)::value, INTERP>(
        grad_out, img, pix, aptr, arg, grad_fmap, B, C, H, W, Vw, P, mw1, mh1, workspace, st);
  });
}

extern "C" size_t dva_gather_pool_bwd_det_workspace_bytes(int64_t B, int64_t H, int64_t W, int64_t P) {
  return det::workspace_bytes(B, H, W, P, 1);
}

extern "C" int dva_gather_pool_bwd_det(const void* grad_out, int channels_last, const int64_t* img,
                                       const void* pix, int pix_is_i16, const int64_t* aptr,
                                       const int64_t* arg, float* grad_fmap, int64_t B, int64_t C,
                                       int64_t H, int64_t W, int64_t Vw, int64_t P, int reduce,
                                       int dtype, void* workspace, size_t workspace_bytes, void* stream) {
  return gather_pool_bwd_det_impl<false>("gather_pool_bwd_det", grad_out, channels_last, img, pix, pix_is_i16,
                                         aptr, arg, grad_fmap, B, C, H, W, 0, 0, Vw, P, reduce, dtype, workspace,
                                         workspace_bytes, stream);
}

extern "C" size_t dva_interp_pool_bwd_det_workspace_bytes(int64_t B, int64_t H, int64_t W, int64_t P) {
  return det::workspace_bytes(B, H, W, P, 4);
}

extern "C" int dva_interp_pool_bwd_det(const void* grad_out, int channels_last, const int64_t* img,
                                       const void* pix, int pix_is_i16, const int64_t* aptr,
                                       const int64_t* arg, float* grad_fmap, int64_t B, int64_t C,
                                       int64_t H, int64_t W, int64_t map_w, int64_t map_h, int64_t Vw,
                                       int64_t P, int reduce, int dtype, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  return gather_pool_bwd_det_impl<true>("interp_pool_bwd_det", grad_out, channels_last, img, pix, pix_is_i16,
                                        aptr, arg, grad_fmap, B, C, H, W, map_w, map_h, Vw, P, reduce, dtype,
                                        workspace, workspace_bytes, stream);
}

// ---------------------------------------------------------------------------------------------
// [B, R, S] -> [B, S, R] (NCHW <-> NHWC with R = C, S = H*W or the reverse): lets the reference's
// NCHW-contiguous feature maps use the channels-last gather / scatter kernels when a large share of
// the map is gathered.  32 x 32 shared tiles, both sides coalesced.
// ---------------------------------------------------------------------------------------------
namespace dva {
template <typename T>
__global__ void __launch_bounds__(256)
transpose_last2_kernel(const T* __restrict__ src, T* __restrict__ dst, int64_t R, int64_t S) {
  __shared__ T tile[32][33];
  const int64_t b = blockIdx.z;
  const int64_t s0 = (int64_t)blockIdx.x * 32, r0 = (int64_t)blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // 32 x 8 threads
  const T* sb = src + b * R * S;
  T* db = dst + b * R * S;
#pragma unroll
  for (int j = 0; j < 32; j += 8) {
    const int64_t r = r0 + ty + j, s = s0 + tx;
    if (r < R && s < S) tile[ty + j][tx] = sb[r * S + s];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 32; j += 8) {
    const int64_t s = s0 + ty + j, r = r0 + tx;
    if (r < R && s < S) db[s * R + r] = tile[tx][ty + j];
  }
}
}  // namespace dva

extern "C" int dva_transpose_last2(const void* src, void* dst, int64_t B, int64_t R, int64_t S, int dtype,
                                   void* stream) {
  if (B < 0 || R < 0 || S < 0) return fail(DVA_EINVAL, "transpose_last2: negative size");
  if (B == 0 || R == 0 || S == 0) return DVA_OK;
  if (!src || !dst) return fail(DVA_EINVAL, "transpose_last2: null pointer");
  if (B > 65535 || (R + 31) / 32 > 65535) return fail(DVA_EUNSUPPORTED, "transpose_last2: batch / row count too large");
  const dim3 grid((unsigned)((S + 31) / 32), (unsigned)((R + 31) / 32), (unsigned)B);
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "transpose_last2: unknown dtype");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DVA_F32)   // bf16 and fp16 move as the same 2-byte words
    transpose_last2_kernel<float><<<grid, 256, 0, st>>>((const float*)src, (float*)dst, R, S);
  else
    transpose_last2_kernel<uint16_t><<<grid, 256, 0, st>>>((const uint16_t*)src, (uint16_t*)dst, R, S);
  return check_launch("transpose_last2");
}
