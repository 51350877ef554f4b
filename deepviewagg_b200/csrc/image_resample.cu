// Image loading on the GPU (SameSettingImageData.read_images / NonStaticMask, core/multimodal/image.py):
//
//   dva_resample_u8      Pillow's 8-bit two-pass convolution resize (ImagingResample with the BICUBIC
//                        filter), batched over B channels-last uint8 images, bit-exact
//   dva_nonstatic_mask   the pixels that differ in every channel between image 0 and some image i >= 1
//
// The coefficient tables come from the caller (ops.resample_tables): int32 weights already scaled by
// 2^22 and rounded as Pillow rounds them, so the kernels are pure integer arithmetic.
#include "dva_common.cuh"

namespace dva {

static constexpr int kPrecisionBits = 32 - 8 - 2;

// Pillow's clip8: the sum carries a +2^21 rounding term; >> 22, clamped to [0, 255]
__device__ __forceinline__ uint8_t clip8(int32_t s) {
  const int32_t v = s >> kPrecisionBits;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Horizontal pass: one thread per output pixel (all channels) of rows t < T of image b, source row
// yfirst_b + t.  Reads the bounds[1] contiguous source pixels from bounds[0] on.
template <int C>
static __global__ void __launch_bounds__(256)
resample_h_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ dst, int64_t B, int64_t Hi, int64_t Wi,
                  int64_t T, int64_t Wo, const int32_t* __restrict__ bounds, const int32_t* __restrict__ coef,
                  int64_t k, int per_image, const int32_t* __restrict__ yfirst) {
  const int64_t total = B * T * Wo;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t x = i % Wo, r = i / Wo, t = r % T, b = r / T;
    const int64_t y = (yfirst ? yfirst[b] : 0) + t;
    if (y >= Hi) continue;                                   // past this image's last used row
    const int64_t e = (per_image ? b * Wo : 0) + x;
    const int32_t xmin = bounds[2 * e], xn = bounds[2 * e + 1];
    const int32_t* kk = coef + e * k;
    const uint8_t* src = in + ((b * Hi + y) * Wi + xmin) * C;
    int32_t s[C];
#pragma unroll
    for (int c = 0; c < C; ++c) s[c] = 1 << (kPrecisionBits - 1);
    for (int32_t j = 0; j < xn; ++j) {
      const int32_t w = __ldg(kk + j);
#pragma unroll
      for (int c = 0; c < C; ++c) s[c] += (int32_t)src[j * C + c] * w;
    }
    uint8_t* o = dst + i * C;
#pragma unroll
    for (int c = 0; c < C; ++c) o[c] = clip8(s[c]);
  }
}

// Vertical pass: one thread per output pixel; the bounds[1] source rows are strided by the row pitch and
// coalesced across x.
template <int C>
static __global__ void __launch_bounds__(256)
resample_v_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ out, int64_t B, int64_t Hs, int64_t W,
                  int64_t Ho, const int32_t* __restrict__ bounds, const int32_t* __restrict__ coef, int64_t k,
                  int per_image) {
  const int64_t total = B * Ho * W, pitch = W * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t x = i % W, r = i / W, yo = r % Ho, b = r / Ho;
    const int64_t e = (per_image ? b * Ho : 0) + yo;
    const int32_t ymin = bounds[2 * e], yn = bounds[2 * e + 1];
    const int32_t* kk = coef + e * k;
    const uint8_t* p = src + ((b * Hs + ymin) * W + x) * C;
    int32_t s[C];
#pragma unroll
    for (int c = 0; c < C; ++c) s[c] = 1 << (kPrecisionBits - 1);
    for (int32_t j = 0; j < yn; ++j) {
      const int32_t w = __ldg(kk + j);
#pragma unroll
      for (int c = 0; c < C; ++c) s[c] += (int32_t)p[j * pitch + c] * w;
    }
    uint8_t* o = out + i * C;
#pragma unroll
    for (int c = 0; c < C; ++c) o[c] = clip8(s[c]);
  }
}

// mask[x, y] (x-major) = OR over i >= 1 of AND over c of (img_i[y, x, c] != img_0[y, x, c]); one thread per
// pixel, x fastest so that the image reads coalesce.
template <int C>
static __global__ void __launch_bounds__(256)
nonstatic_mask_kernel(const uint8_t* __restrict__ imgs, int64_t n, int64_t H, int64_t W, uint8_t* __restrict__ mask) {
  const int64_t HW = H * W;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t y = i / W, x = i - y * W;
    uint8_t ref[C];
#pragma unroll
    for (int c = 0; c < C; ++c) ref[c] = imgs[i * C + c];
    bool any = false;
    for (int64_t m = 1; m < n && !any; ++m) {
      const uint8_t* p = imgs + (m * HW + i) * C;
      bool all = true;
#pragma unroll
      for (int c = 0; c < C; ++c) all = all && (p[c] != ref[c]);
      any = all;
    }
    mask[x * H + y] = any ? 1 : 0;
  }
}

template <int C>
static int resample_launch(const uint8_t* in, uint8_t* tmp, uint8_t* out, int64_t B, int64_t Hi, int64_t Wi,
                           int64_t Ho, int64_t Wo, int64_t T, const int32_t* xb, const int32_t* xc, int64_t kx,
                           int xpi, const int32_t* yb, const int32_t* yc, int64_t ky, int ypi, const int32_t* yfirst,
                           cudaStream_t st) {
  if (xc) {
    uint8_t* dst = yc ? tmp : out;
    resample_h_kernel<C><<<grid_cap(B * T * Wo, 256, 16), 256, 0, st>>>(in, dst, B, Hi, Wi, T, Wo, xb, xc, kx, xpi, yfirst);
    const int rc = check_launch("resample_u8_horizontal");
    if (rc) return rc;
  }
  if (yc) {
    const uint8_t* src = xc ? tmp : in;
    const int64_t Hs = xc ? T : Hi;
    resample_v_kernel<C><<<grid_cap(B * Ho * Wo, 256, 16), 256, 0, st>>>(src, out, B, Hs, Wo, Ho, yb, yc, ky, ypi);
    return check_launch("resample_u8_vertical");
  }
  return DVA_OK;
}

}  // namespace dva

using namespace dva;

extern "C" int dva_resample_u8(const uint8_t* in, uint8_t* tmp, uint8_t* out, int64_t B, int64_t Hi, int64_t Wi,
                               int64_t C, int64_t Ho, int64_t Wo, int64_t T, const int32_t* xbounds,
                               const int32_t* xcoef, int64_t kx, int x_per_image, const int32_t* ybounds,
                               const int32_t* ycoef, int64_t ky, int y_per_image, const int32_t* yfirst,
                               void* stream) {
  if (B < 0 || Hi < 0 || Wi < 0 || Ho < 0 || Wo < 0 || T < 0) return fail(DVA_EINVAL, "resample_u8: negative size");
  if (C < 1 || C > 4) return fail(DVA_EUNSUPPORTED, "resample_u8: 1 to 4 channels");
  if (!xcoef && !ycoef) return fail(DVA_EINVAL, "resample_u8: neither pass requested");
  if (xcoef && (!xbounds || kx < 1)) return fail(DVA_EINVAL, "resample_u8: horizontal table missing");
  if (ycoef && (!ybounds || ky < 1)) return fail(DVA_EINVAL, "resample_u8: vertical table missing");
  if (!xcoef && Wo != Wi) return fail(DVA_EINVAL, "resample_u8: a vertical-only resize keeps the width");
  if (xcoef && ycoef && (!tmp || T < 1)) return fail(DVA_EINVAL, "resample_u8: two passes need a temporary");
  if (xcoef && !ycoef && T != Ho) return fail(DVA_EINVAL, "resample_u8: a horizontal-only resize writes Ho rows");
  if (B == 0 || Ho == 0 || Wo == 0) return DVA_OK;
  if (Hi == 0 || Wi == 0) return fail(DVA_EINVAL, "resample_u8: empty input");
  if (!in || !out) return fail(DVA_EINVAL, "resample_u8: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  switch (C) {
    case 1: return resample_launch<1>(in, tmp, out, B, Hi, Wi, Ho, Wo, T, xbounds, xcoef, kx, x_per_image, ybounds,
                                      ycoef, ky, y_per_image, yfirst, st);
    case 2: return resample_launch<2>(in, tmp, out, B, Hi, Wi, Ho, Wo, T, xbounds, xcoef, kx, x_per_image, ybounds,
                                      ycoef, ky, y_per_image, yfirst, st);
    case 3: return resample_launch<3>(in, tmp, out, B, Hi, Wi, Ho, Wo, T, xbounds, xcoef, kx, x_per_image, ybounds,
                                      ycoef, ky, y_per_image, yfirst, st);
    default: return resample_launch<4>(in, tmp, out, B, Hi, Wi, Ho, Wo, T, xbounds, xcoef, kx, x_per_image, ybounds,
                                       ycoef, ky, y_per_image, yfirst, st);
  }
}

extern "C" int dva_nonstatic_mask(const uint8_t* imgs, int64_t n, int64_t H, int64_t W, int64_t C, uint8_t* mask,
                                  void* stream) {
  if (n < 2) return fail(DVA_EINVAL, "nonstatic_mask: needs at least 2 images");
  if (H < 0 || W < 0) return fail(DVA_EINVAL, "nonstatic_mask: negative size");
  if (C < 1 || C > 4) return fail(DVA_EUNSUPPORTED, "nonstatic_mask: 1 to 4 channels");
  if (H == 0 || W == 0) return DVA_OK;
  if (!imgs || !mask) return fail(DVA_EINVAL, "nonstatic_mask: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_cap(H * W, 256, 16);
  switch (C) {
    case 1: nonstatic_mask_kernel<1><<<g, 256, 0, st>>>(imgs, n, H, W, mask); break;
    case 2: nonstatic_mask_kernel<2><<<g, 256, 0, st>>>(imgs, n, H, W, mask); break;
    case 3: nonstatic_mask_kernel<3><<<g, 256, 0, st>>>(imgs, n, H, W, mask); break;
    default: nonstatic_mask_kernel<4><<<g, 256, 0, st>>>(imgs, n, H, W, mask); break;
  }
  return check_launch("nonstatic_mask");
}
