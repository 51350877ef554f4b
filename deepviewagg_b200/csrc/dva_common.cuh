// Shared device/host helpers for libdva_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <type_traits>
#include "../../include/dva_b200.h"

namespace dva {

constexpr int kNumSMs = 132;  // H100 SXM; grids are sized in multiples of this

// ---- thread-local error string + launch counter (C ABI: dva_last_error), process-wide launch counter (dva_launch_count)
char* tls_error_buf();
std::atomic<int64_t>& launch_counter();

inline int fail(int code, const char* msg) {
  snprintf(tls_error_buf(), 256, "%s", msg);
  return code;
}

template <typename... A> inline int failf(int code, const char* fmt, A... a) {
  snprintf(tls_error_buf(), 256, fmt, a...);
  return code;
}

inline int check_launch(const char* what) {
  launch_counter().fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    snprintf(tls_error_buf(), 256, "%s: %s", what, cudaGetErrorString(e));
    return (int)e;
  }
  return DVA_OK;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- host-side launch vocabulary: every launcher takes these decisions from here
// f(T{}) with T the storage type of dtype; the C entry points have rejected every other dtype
template <typename F> decltype(auto) with_dtype(int dtype, F&& f) {
  switch (dtype) {
    case DVA_F32: return f(float{});
    case DVA_BF16: return f(__nv_bfloat16{});
    default: return f(__half{});
  }
}
inline bool known_dtype(int dtype) { return dtype == DVA_F32 || dtype == DVA_BF16 || dtype == DVA_F16; }

// f(std::integral_constant<int, V>{}) for the V of Vs equal to v; false (f not called) when there is none
template <int... Vs, typename F> bool with_value(int v, F&& f) {
  return ((v == Vs && (f(std::integral_constant<int, Vs>{}), true)) || ...);
}
// f(std::integral_constant<int, RED>{}) with RED the reduce code; false for an unknown code
template <typename F> bool with_reduce(int reduce, F&& f) {
  return with_value<DVA_SUM, DVA_MEAN, DVA_MAX, DVA_MIN>(reduce, f);
}
// f(PIX{}) with PIX the type of the (x, y) pixel pairs of pix_code 0 = int16, 1 = int32, 2 = int64; false for any
// other code
template <typename F> bool with_pix(int pix_code, F&& f) {
  return with_value<0, 1, 2>(pix_code, [&](auto c) {
    constexpr int k = decltype(c)::value;
    f(std::conditional_t<k == 0, int16_t, std::conditional_t<k == 1, int32_t, int64_t>>{});
  });
}
// f(std::integral_constant<int, LPR>{}) with LPR the lanes per row of the sub-warp row kernels: the smallest of
// 4, 8, 16, 32 that covers cv 16-byte chunks
template <typename F> decltype(auto) with_lpr(int64_t cv, F&& f) {
  if (cv <= 4) return f(std::integral_constant<int, 4>{});
  if (cv <= 8) return f(std::integral_constant<int, 8>{});
  if (cv <= 16) return f(std::integral_constant<int, 16>{});
  return f(std::integral_constant<int, 32>{});
}

// Grid of a grid-stride launch: one CTA per per_block items, at least 1 and at most ctas_per_sm CTAs per SM
inline int grid_cap(int64_t items, int64_t per_block, int ctas_per_sm) {
  const int64_t blocks = (items + per_block - 1) / per_block, cap = (int64_t)kNumSMs * ctas_per_sm;
  return (int)(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
}

// workspaces are carved in 256-byte aligned pieces from a 256-byte aligned base
inline size_t round256(size_t bytes) { return (bytes + 255) & ~(size_t)255; }
inline uint8_t* align256(void* p) { return reinterpret_cast<uint8_t*>(round256(reinterpret_cast<uintptr_t>(p))); }

// the opt-in a kernel needs to launch with more than 48 KB of dynamic shared memory
template <typename K> cudaError_t smem_opt_in(K* kern, size_t smem) {
  if (smem <= 48 * 1024) return cudaSuccess;
  return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

// ---- storage-type traits: load/store as fp32
template <typename T> struct Cvt;
template <> struct Cvt<float> {
  static __device__ __forceinline__ float to_f(float v) { return v; }
  static __device__ __forceinline__ float from_f(float v) { return v; }
};
template <> struct Cvt<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <> struct Cvt<__half> {
  static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};

// 16-byte vector of T: float x4, bf16/half x8
template <typename T> struct Vec16 { static constexpr int N = 16 / sizeof(T); };

// rows of n elements of T can move as 16-byte vectors: n is a multiple of Vec16<T>::N and every pointer is
// 16-byte aligned (a null pointer, an absent operand, counts as aligned)
template <typename T, typename... P> bool vec16_ok(int64_t n, const P*... p) {
  return n % Vec16<T>::N == 0 && (aligned16(p) && ...);
}

template <typename T, int N>
struct alignas(sizeof(T) * N) Pack { T v[N]; };

// streaming 16-byte load/store (rows are touched once: keep them out of L1)
__device__ __forceinline__ uint4 ldg_stream16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void stg_stream16(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// 16-byte vector reduction into global memory (sm_90+): one instruction per four channels
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

template <typename T, int VEC>
__device__ __forceinline__ void unpack16(const uint4& raw, float (&f)[VEC]);
template <> __device__ __forceinline__ void unpack16<float, 4>(const uint4& raw, float (&f)[4]) {
  f[0] = __uint_as_float(raw.x); f[1] = __uint_as_float(raw.y);
  f[2] = __uint_as_float(raw.z); f[3] = __uint_as_float(raw.w);
}
template <> __device__ __forceinline__ void unpack16<__nv_bfloat16, 8>(const uint4& raw, float (&f)[8]) {
  const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {  // bf16 -> fp32 is a 16-bit shift
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}
template <> __device__ __forceinline__ void unpack16<__half, 8>(const uint4& raw, float (&f)[8]) {
  const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
    float2 t = __half22float2(h);
    f[2 * i] = t.x; f[2 * i + 1] = t.y;
  }
}

template <typename T, int VEC>
__device__ __forceinline__ uint4 pack16(const float (&f)[VEC]);
template <> __device__ __forceinline__ uint4 pack16<float, 4>(const float (&f)[4]) {
  return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                    __float_as_uint(f[3]));
}
template <> __device__ __forceinline__ uint4 pack16<__nv_bfloat16, 8>(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
template <> __device__ __forceinline__ uint4 pack16<__half, 8>(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// channel -> group of pooling.py:737-755 (group_sizes / expand_group_feat):
// sizes floor(C/G), the first C%G groups one wider.
__host__ __device__ __forceinline__ int group_of_channel(int c, int C, int G) {
  const int base = C / G, rem = C - base * G;
  const int wide = rem * (base + 1);
  return c < wide ? c / (base + 1) : rem + (c - wide) / base;
}

__device__ __forceinline__ int64_t load_idx(const void* idx, bool is64, int64_t v) {
  if (idx == nullptr) return v;
  return is64 ? reinterpret_cast<const int64_t*>(idx)[v]
              : (int64_t) reinterpret_cast<const int32_t*>(idx)[v];
}

}  // namespace dva
