// Colour transforms of a loaded sample (core/multimodal/transforms.py: ColorJitter, ToFloatImage, Normalize):
//
//   dva_color_jitter_u8   torchvision's ColorJitter (brightness, contrast, saturation; no hue) on [B, 3, H, W]
//                         uint8 with drawn factors, every op of the drawn order in one pass over the pixels
//   dva_image_to_float    (x - m_c) / s_c in fp32 with true division: ToFloatImage (m = 0, s = 255, uint8 in)
//                         and Normalize (fp32 in)
//
// The fp32 arithmetic restates torchvision's _functional_tensor op by op (oracle/color_oracle.py): products
// and sums are __fmul_rn / __fadd_rn (no FMA contraction), sums run left to right, a blend is clamped to
// [0, 255] and truncated to uint8 after every op.  The contrast mean is float32(float64(S) / float64(H W)) of
// the exact integer sum S of the grayscale bytes, so it does not depend on the launch.
#include "dva_common.cuh"

namespace dva {

enum { kBrightness = 0, kContrast = 1, kSaturation = 2 };

struct JitterOps {
  int n;          // active ops, applied in order
  int code[3];    // kBrightness / kContrast / kSaturation
  float ratio[3];
  float rest[3];  // fp32(1 - ratio), rounded from float64 on the host
};

// torchvision rgb_to_grayscale: (0.2989 r + 0.587 g) + 0.114 b in fp32, truncated to uint8
__device__ __forceinline__ uint32_t gray_u8(uint32_t r, uint32_t g, uint32_t b) {
  const float l = __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, (float)r), __fmul_rn(0.587f, (float)g)),
                            __fmul_rn(0.114f, (float)b));
  return __float2uint_rz(l);
}

// torchvision _blend for uint8: fp32(ratio) * v + other_term, clamped to [0, 255], truncated
__device__ __forceinline__ uint32_t blend_u8(uint32_t v, float ratio, float other_term) {
  const float f = __fadd_rn(__fmul_rn(ratio, (float)v), other_term);
  return __float2uint_rz(fminf(fmaxf(f, 0.f), 255.f));
}

// ops [first, last) of the drawn order on one pixel; `mean` is the contrast mean of the pixel's image
__device__ __forceinline__ void apply_ops(const JitterOps& ops, int first, int last, float mean, uint32_t& r,
                                          uint32_t& g, uint32_t& b) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < first || i >= last) continue;
    const float ra = ops.ratio[i], re = ops.rest[i];
    float other_r, other_g, other_b;
    if (ops.code[i] == kBrightness) {
      other_r = other_g = other_b = __fmul_rn(re, 0.f);       // (1 - ratio) * zeros_like(img)
    } else if (ops.code[i] == kContrast) {
      other_r = other_g = other_b = __fmul_rn(re, mean);
    } else {
      other_r = other_g = other_b = __fmul_rn(re, (float)gray_u8(r, g, b));
    }
    r = blend_u8(r, ra, other_r);
    g = blend_u8(g, ra, other_g);
    b = blend_u8(b, ra, other_b);
  }
}

// Pixels of image b: [0, head) and [head + 16 n_vec, HW) one at a time, [head, head + 16 n_vec) as chunks of
// 16 pixels loaded and stored 16 bytes wide.  Channels-last: a chunk is 48 contiguous bytes, aligned when its
// first pixel is a multiple of 16 of the whole batch.  NCHW: a chunk is 16 bytes of each plane, aligned for
// every chunk only when HW % 16 == 0; otherwise every pixel goes one at a time.
struct Span {
  int64_t head, n_vec;
};
__device__ __forceinline__ Span image_span(int64_t b, int64_t HW, bool cl, bool vec_ok) {
  Span s{HW, 0};
  if (!vec_ok) return s;
  if (cl) {
    const int64_t lead = (16 - (b * HW) % 16) % 16;
    s.head = lead < HW ? lead : HW;
  } else {
    if (HW % 16 != 0) return s;
    s.head = 0;
  }
  s.n_vec = (HW - s.head) / 16;
  return s;
}

__device__ __forceinline__ uint32_t byte_of(const uint4& v, int i) {
  const uint32_t w = i < 4 ? v.x : (i < 8 ? v.y : (i < 12 ? v.z : v.w));
  return (w >> (8 * (i & 3))) & 0xffu;
}
__device__ __forceinline__ void set_byte(uint4& v, int i, uint32_t byte) {
  uint32_t& w = i < 4 ? v.x : (i < 8 ? v.y : (i < 12 ? v.z : v.w));
  const int sh = 8 * (i & 3);
  w = (w & ~(0xffu << sh)) | (byte << sh);
}

// byte offset of channel c of pixel p of image b
__device__ __forceinline__ int64_t chan_off(int64_t b, int64_t p, int c, int64_t HW, bool cl) {
  return cl ? (b * HW + p) * 3 + c : (b * 3 + c) * HW + p;
}

__device__ __forceinline__ float image_mean(const unsigned long long* sums, int64_t b, int64_t HW) {
  return __double2float_rn(__ddiv_rn((double)sums[b], (double)HW));
}

// Sum pass: sums[b] += the grayscale bytes of image b after the ops before contrast (ops [0, upto)).  Per-thread
// integer partials, a warp reduction, one 64-bit atomic per warp per image (sums zeroed by the caller).
static __global__ void __launch_bounds__(256)
jitter_sum_kernel(const uint8_t* __restrict__ in, int64_t B, int64_t HW, int cl, int vec_ok, JitterOps ops, int upto,
                  unsigned long long* __restrict__ sums) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, nthr = (int64_t)gridDim.x * blockDim.x;
  for (int64_t b = blockIdx.y; b < B; b += gridDim.y) {
    const Span s = image_span(b, HW, cl, vec_ok);
    unsigned long long acc = 0;
    for (int64_t k = tid; k < s.n_vec; k += nthr) {
      const int64_t p0 = s.head + 16 * k;
      uint32_t part = 0;
      if (cl) {
        const uint8_t* src = in + (b * HW + p0) * 3;
        const uint4 v0 = ldg_stream16(src), v1 = ldg_stream16(src + 16), v2 = ldg_stream16(src + 32);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          uint32_t ch[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const int i = 3 * j + c;
            ch[c] = byte_of(i < 16 ? v0 : (i < 32 ? v1 : v2), i & 15);
          }
          apply_ops(ops, 0, upto, 0.f, ch[0], ch[1], ch[2]);
          part += gray_u8(ch[0], ch[1], ch[2]);
        }
      } else {
        const uint8_t* src = in + b * 3 * HW + p0;
        const uint4 vr = ldg_stream16(src), vg = ldg_stream16(src + HW), vb = ldg_stream16(src + 2 * HW);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          uint32_t r = byte_of(vr, j), g = byte_of(vg, j), bl = byte_of(vb, j);
          apply_ops(ops, 0, upto, 0.f, r, g, bl);
          part += gray_u8(r, g, bl);
        }
      }
      acc += part;
    }
    const int64_t n_scalar = HW - 16 * s.n_vec;
    for (int64_t k = tid; k < n_scalar; k += nthr) {
      const int64_t p = k < s.head ? k : k + 16 * s.n_vec;
      uint32_t r = in[chan_off(b, p, 0, HW, cl)], g = in[chan_off(b, p, 1, HW, cl)], bl = in[chan_off(b, p, 2, HW, cl)];
      apply_ops(ops, 0, upto, 0.f, r, g, bl);
      acc += gray_u8(r, g, bl);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc != 0) atomicAdd(sums + b, acc);
  }
}

// Apply pass: every op of the drawn order on every pixel; the contrast mean is read from sums on the device.
static __global__ void __launch_bounds__(256)
jitter_apply_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int64_t B, int64_t HW, int cl,
                    int vec_ok, JitterOps ops, const unsigned long long* __restrict__ sums) {
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, nthr = (int64_t)gridDim.x * blockDim.x;
  for (int64_t b = blockIdx.y; b < B; b += gridDim.y) {
    const Span s = image_span(b, HW, cl, vec_ok);
    const float mean = sums ? image_mean(sums, b, HW) : 0.f;
    for (int64_t k = tid; k < s.n_vec; k += nthr) {
      const int64_t p0 = s.head + 16 * k;
      if (cl) {
        const int64_t off = (b * HW + p0) * 3;
        uint4 v[3] = {ldg_stream16(in + off), ldg_stream16(in + off + 16), ldg_stream16(in + off + 32)};
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          uint32_t ch[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) ch[c] = byte_of(v[(3 * j + c) >> 4], (3 * j + c) & 15);
          apply_ops(ops, 0, ops.n, mean, ch[0], ch[1], ch[2]);
#pragma unroll
          for (int c = 0; c < 3; ++c) set_byte(v[(3 * j + c) >> 4], (3 * j + c) & 15, ch[c]);
        }
        stg_stream16(out + off, v[0]);
        stg_stream16(out + off + 16, v[1]);
        stg_stream16(out + off + 32, v[2]);
      } else {
        const int64_t off = b * 3 * HW + p0;
        uint4 vr = ldg_stream16(in + off), vg = ldg_stream16(in + off + HW), vb = ldg_stream16(in + off + 2 * HW);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          uint32_t r = byte_of(vr, j), g = byte_of(vg, j), bl = byte_of(vb, j);
          apply_ops(ops, 0, ops.n, mean, r, g, bl);
          set_byte(vr, j, r);
          set_byte(vg, j, g);
          set_byte(vb, j, bl);
        }
        stg_stream16(out + off, vr);
        stg_stream16(out + off + HW, vg);
        stg_stream16(out + off + 2 * HW, vb);
      }
    }
    const int64_t n_scalar = HW - 16 * s.n_vec;
    for (int64_t k = tid; k < n_scalar; k += nthr) {
      const int64_t p = k < s.head ? k : k + 16 * s.n_vec;
      const int64_t o0 = chan_off(b, p, 0, HW, cl), o1 = chan_off(b, p, 1, HW, cl), o2 = chan_off(b, p, 2, HW, cl);
      uint32_t r = in[o0], g = in[o1], bl = in[o2];
      apply_ops(ops, 0, ops.n, mean, r, g, bl);
      out[o0] = (uint8_t)r;
      out[o1] = (uint8_t)g;
      out[o2] = (uint8_t)bl;
    }
  }
}

struct ChannelStats {
  float m[4], s[4];
};

// (x - m_c) / s_c; the channel is picked by selects so that the kernel parameters stay out of local memory
__device__ __forceinline__ float normalize_one(float x, const ChannelStats& st, int c) {
  const float m = c == 0 ? st.m[0] : (c == 1 ? st.m[1] : (c == 2 ? st.m[2] : st.m[3]));
  const float s = c == 0 ? st.s[0] : (c == 1 ? st.s[1] : (c == 2 ? st.s[2] : st.s[3]));
  return __fdiv_rn(__fsub_rn(x, m), s);
}

// out = (x - m_c) / s_c, one element per thread; NCHW: c = (i / HW) % C, channels-last: c = i % C
template <typename Tin>
static __global__ void __launch_bounds__(256)
to_float_kernel(const Tin* __restrict__ in, float* __restrict__ out, int64_t total, int64_t HW, int C, int cl,
                ChannelStats st) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = cl ? (int)(i % C) : (int)((i / HW) % C);
    out[i] = normalize_one((float)in[i], st, c);
  }
}

// the same with 16-byte loads and stores: 16 uint8 or 4 fp32 in, 16 / 4 fp32 out per step
template <typename Tin>
static __global__ void __launch_bounds__(256)
to_float_vec_kernel(const Tin* __restrict__ in, float* __restrict__ out, int64_t total, int64_t HW, int C, int cl,
                    ChannelStats st) {
  constexpr int V = 16 / sizeof(Tin);
  const int64_t nv = total / V;
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nv; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i0 = k * V;
    const uint4 raw = ldg_stream16(in + i0);
    float f[V];
    if constexpr (sizeof(Tin) == 1) {
#pragma unroll
      for (int j = 0; j < 16; ++j) f[j] = (float)byte_of(raw, j);
    } else {
      f[0] = __uint_as_float(raw.x); f[1] = __uint_as_float(raw.y);
      f[2] = __uint_as_float(raw.z); f[3] = __uint_as_float(raw.w);
    }
    // channels-last: the channel cycles along the chunk; NCHW: HW % 16 == 0, so the chunk lies in one plane
    int c = cl ? (int)(i0 % C) : (int)((i0 / HW) % C);
#pragma unroll
    for (int j = 0; j < V; ++j) {
      f[j] = normalize_one(f[j], st, c);
      if (cl) c = c + 1 == C ? 0 : c + 1;
    }
#pragma unroll
    for (int j = 0; j < V; j += 4)
      stg_stream16(out + i0 + j, make_uint4(__float_as_uint(f[j]), __float_as_uint(f[j + 1]),
                                            __float_as_uint(f[j + 2]), __float_as_uint(f[j + 3])));
  }
}

}  // namespace dva

using namespace dva;

extern "C" size_t dva_color_jitter_u8_workspace_bytes(int64_t B) {
  return B > 0 ? (size_t)B * sizeof(unsigned long long) : 0;
}

extern "C" int dva_color_jitter_u8(const uint8_t* in, uint8_t* out, int64_t B, int64_t H, int64_t W,
                                   int channels_last, int n_ops, int op_codes, float ratio0, float rest0, float ratio1,
                                   float rest1, float ratio2, float rest2, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  if (B < 0 || H < 0 || W < 0) return fail(DVA_EINVAL, "color_jitter_u8: negative size");
  if (n_ops < 0 || n_ops > 3) return fail(DVA_EINVAL, "color_jitter_u8: 0 to 3 ops");
  JitterOps ops;
  ops.n = n_ops;
  const float ratio[3] = {ratio0, ratio1, ratio2}, rest[3] = {rest0, rest1, rest2};
  int seen = 0, contrast_at = -1;
  for (int i = 0; i < 3; ++i) {
    ops.code[i] = (op_codes >> (4 * i)) & 0xf;
    ops.ratio[i] = ratio[i];
    ops.rest[i] = rest[i];
    if (i >= n_ops) continue;
    if (ops.code[i] > kSaturation) return fail(DVA_EINVAL, "color_jitter_u8: op code must be 0, 1 or 2");
    if (seen & (1 << ops.code[i])) return fail(DVA_EINVAL, "color_jitter_u8: an op appears twice");
    if (!(ratio[i] >= 0.f)) return fail(DVA_EINVAL, "color_jitter_u8: factors must be non negative");
    seen |= 1 << ops.code[i];
    if (ops.code[i] == kContrast) contrast_at = i;
  }
  if (contrast_at >= 0 && (!workspace || workspace_bytes < dva_color_jitter_u8_workspace_bytes(B)))
    return fail(DVA_EINVAL, "color_jitter_u8: workspace too small (dva_color_jitter_u8_workspace_bytes)");
  const int64_t HW = H * W;
  if (B == 0 || HW == 0) return DVA_OK;
  if (!in || !out) return fail(DVA_EINVAL, "color_jitter_u8: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int cl = channels_last != 0;
  const int vec_ok = aligned16(in) && aligned16(out);
  // blocks per image: 16-pixel chunks over 256 threads, all images together within the grid cap
  const int64_t per_img = (HW / 16 + 255) / 256, cap = (int64_t)kNumSMs * 16;
  const int64_t by = B < 65535 ? B : 65535;
  int64_t bx = per_img < 1 ? 1 : per_img;
  if (bx * by > cap) bx = cap / by > 0 ? cap / by : 1;
  const dim3 grid((unsigned)bx, (unsigned)by);
  unsigned long long* sums = nullptr;
  if (contrast_at >= 0) {
    sums = (unsigned long long*)workspace;
    const cudaError_t e = cudaMemsetAsync(sums, 0, (size_t)B * sizeof(unsigned long long), st);
    if (e != cudaSuccess) return failf((int)e, "color_jitter_u8: memset: %s", cudaGetErrorString(e));
    jitter_sum_kernel<<<grid, 256, 0, st>>>(in, B, HW, cl, vec_ok, ops, contrast_at, sums);
    const int rc = check_launch("color_jitter_u8_sum");
    if (rc) return rc;
  }
  jitter_apply_kernel<<<grid, 256, 0, st>>>(in, out, B, HW, cl, vec_ok, ops, sums);
  return check_launch("color_jitter_u8_apply");
}

extern "C" int dva_image_to_float(const void* in, int in_u8, float* out, int64_t B, int64_t C, int64_t H, int64_t W,
                                  int channels_last, float m0, float m1, float m2, float m3, float s0, float s1,
                                  float s2, float s3, void* stream) {
  if (B < 0 || H < 0 || W < 0) return fail(DVA_EINVAL, "image_to_float: negative size");
  if (C < 1 || C > 4) return fail(DVA_EUNSUPPORTED, "image_to_float: 1 to 4 channels");
  const int64_t total = B * C * H * W;
  if (total == 0) return DVA_OK;
  if (!in || !out) return fail(DVA_EINVAL, "image_to_float: null pointer");
  const ChannelStats st{{m0, m1, m2, m3}, {s0, s1, s2, s3}};
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t HW = H * W;
  const int cl = channels_last != 0;
  const bool vec = aligned16(in) && aligned16(out) && total % 16 == 0 && (cl || HW % 16 == 0);
  if (in_u8) {
    const uint8_t* x = (const uint8_t*)in;
    if (vec) to_float_vec_kernel<uint8_t><<<grid_cap(total / 16, 256, 16), 256, 0, s>>>(x, out, total, HW, (int)C, cl, st);
    else to_float_kernel<uint8_t><<<grid_cap(total, 256, 16), 256, 0, s>>>(x, out, total, HW, (int)C, cl, st);
  } else {
    const float* x = (const float*)in;
    if (vec) to_float_vec_kernel<float><<<grid_cap(total / 4, 256, 16), 256, 0, s>>>(x, out, total, HW, (int)C, cl, st);
    else to_float_kernel<float><<<grid_cap(total, 256, 16), 256, 0, s>>>(x, out, total, HW, (int)C, cl, st);
  }
  return check_launch("image_to_float");
}
