// Segmented (CSR) reductions, broadcast and softmax: the building blocks every pool of
// torch_points3d/modules/multimodal/pooling.py composes (segment_csr at :63,:289,:295,:519,:525,
// :628,:787,:807,:851; gather_csr :813-841; segment_softmax_csr :758-810).
//
// Layout: src [n_items,K] row-major, ptr [n_seg+1] int64.  One thread owns one (segment,
// column-vector) pair and walks the segment's rows in order -- adjacent threads own adjacent
// columns, so every row read/write is a coalesced 16-byte-per-lane access, and the reduction
// order is the sequential order of torch_scatter's CPU kernel (deterministic, first arg-max).
// These are HBM-bound streaming kernels: bytes = n_items*K*s (read) + n_seg*K*s (write).
#include "bucket_sort.cuh"

namespace dva {

template <int RED> struct RedOp;
template <> struct RedOp<DVA_SUM> { static __device__ __forceinline__ bool better(float a, float b) { return false; } };
template <> struct RedOp<DVA_MAX> { static __device__ __forceinline__ bool better(float a, float b) { return a > b; } };
template <> struct RedOp<DVA_MIN> { static __device__ __forceinline__ bool better(float a, float b) { return a < b; } };

// Rows outside [ptr[0], ptr[n_seg]) belong to no segment (torch_scatter accepts such pointers): the
// element-level outputs (gradients w.r.t. src, gather_csr / softmax results) are 0 there, never
// uninitialised memory.  Both ranges are empty for a well-formed CSR, so this costs two cached loads.
template <typename T>
__device__ __forceinline__ void zero_uncovered_rows(T* __restrict__ dst, const int64_t* __restrict__ ptr,
                                                    int64_t n_seg, int64_t n_items, int64_t K) {
  const int64_t head = ptr[0] < n_items ? ptr[0] : n_items;
  const int64_t tail0 = ptr[n_seg] > head ? ptr[n_seg] : head;
  const int64_t n_tail = n_items > tail0 ? n_items - tail0 : 0;
  const int64_t total = (head + n_tail) * K;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / K, c = t - r * K;
    const int64_t row = r < head ? r : tail0 + (r - head);
    dst[row * K + c] = Cvt<T>::from_f(0.f);
  }
}

// ---- forward -----------------------------------------------------------------------------
template <typename T, int VEC, int RED>
__global__ void __launch_bounds__(256)
segment_csr_fwd_kernel(const T* __restrict__ src, const int64_t* __restrict__ ptr,
                       T* __restrict__ out, int64_t* __restrict__ arg, int64_t n_seg,
                       int64_t n_items, int64_t K) {
  const int64_t KV = K / VEC;
  const int64_t total = n_seg * KV;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / KV, kv = t - i * KV;
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    float acc[VEC];
    int64_t best[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) { acc[j] = 0.f; best[j] = n_items; }
    const T* col = src + kv * VEC;
    for (int64_t p = p0; p < p1; ++p) {
      Pack<T, VEC> raw = *reinterpret_cast<const Pack<T, VEC>*>(col + p * K);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float v = Cvt<T>::to_f(raw.v[j]);
        if (RED == DVA_SUM || RED == DVA_MEAN) {
          acc[j] += v;
        } else {
          constexpr int R2 = (RED == DVA_MIN) ? DVA_MIN : DVA_MAX;
          if (p == p0 || RedOp<R2>::better(v, acc[j])) { acc[j] = v; best[j] = p; }
        }
      }
    }
    if (RED == DVA_MEAN) {
      const float inv = 1.f / (float)((p1 - p0) > 0 ? (p1 - p0) : 1);
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc[j] *= inv;
    }
    Pack<T, VEC> o;
#pragma unroll
    for (int j = 0; j < VEC; ++j) o.v[j] = Cvt<T>::from_f(acc[j]);
    *reinterpret_cast<Pack<T, VEC>*>(out + i * K + kv * VEC) = o;
    if ((RED == DVA_MAX || RED == DVA_MIN) && arg != nullptr) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) arg[i * K + kv * VEC + j] = best[j];
    }
  }
}

// ---- backward: every row of grad_src is written exactly once (segments partition the rows)
template <typename T, int VEC, int RED>
__global__ void __launch_bounds__(256)
segment_csr_bwd_kernel(const T* __restrict__ gout, const int64_t* __restrict__ ptr,
                       const int64_t* __restrict__ arg, T* __restrict__ gsrc, int64_t n_seg,
                       int64_t n_items, int64_t K) {
  zero_uncovered_rows(gsrc, ptr, n_seg, n_items, K);
  const int64_t KV = K / VEC;
  const int64_t total = n_seg * KV;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / KV, kv = t - i * KV;
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    if (p1 <= p0) continue;
    Pack<T, VEC> g = *reinterpret_cast<const Pack<T, VEC>*>(gout + i * K + kv * VEC);
    int64_t a[VEC];
    if (RED == DVA_MAX || RED == DVA_MIN) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) a[j] = arg[i * K + kv * VEC + j];
    }
    if (RED == DVA_MEAN) {
      const float inv = 1.f / (float)(p1 - p0);
#pragma unroll
      for (int j = 0; j < VEC; ++j) g.v[j] = Cvt<T>::from_f(Cvt<T>::to_f(g.v[j]) * inv);
    }
    for (int64_t p = p0; p < p1; ++p) {
      Pack<T, VEC> o = g;
      if (RED == DVA_MAX || RED == DVA_MIN) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) if (a[j] != p) o.v[j] = Cvt<T>::from_f(0.f);
      }
      *reinterpret_cast<Pack<T, VEC>*>(gsrc + p * K + kv * VEC) = o;
    }
  }
}

// ---- gather_csr: broadcast segment rows to their items
template <typename T, int VEC>
__global__ void __launch_bounds__(256)
gather_csr_kernel(const T* __restrict__ src, const int64_t* __restrict__ ptr,
                  T* __restrict__ out, int64_t n_seg, int64_t n_items, int64_t K) {
  zero_uncovered_rows(out, ptr, n_seg, n_items, K);
  const int64_t KV = K / VEC;
  const int64_t total = n_seg * KV;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / KV, kv = t - i * KV;
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    if (p1 <= p0) continue;
    const Pack<T, VEC> g = *reinterpret_cast<const Pack<T, VEC>*>(src + i * K + kv * VEC);
    for (int64_t p = p0; p < p1; ++p)
      *reinterpret_cast<Pack<T, VEC>*>(out + p * K + kv * VEC) = g;
  }
}

// ---- segment softmax (pooling.py:758-810)
template <typename T>
__global__ void __launch_bounds__(256)
segment_softmax_fwd_kernel(const T* __restrict__ src, const int64_t* __restrict__ ptr,
                           T* __restrict__ out, int64_t n_seg, int64_t n_items, int64_t K, float eps,
                           int scaling) {
  zero_uncovered_rows(out, ptr, n_seg, n_items, K);
  const int64_t total = n_seg * K;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / K, k = t - i * K;
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    if (p1 <= p0) continue;
    float m = Cvt<T>::to_f(src[p0 * K + k]);
    for (int64_t p = p0 + 1; p < p1; ++p) m = fmaxf(m, Cvt<T>::to_f(src[p * K + k]));
    // reference divides the centred score by sqrt(count) (pooling.py:792-801)
    const float sq = scaling ? sqrtf((float)(p1 - p0)) : 1.f;
    float sum = 0.f;
    for (int64_t p = p0; p < p1; ++p) sum += expf((Cvt<T>::to_f(src[p * K + k]) - m) / sq);
    const float den = sum + eps;
    for (int64_t p = p0; p < p1; ++p)
      out[p * K + k] = Cvt<T>::from_f(expf((Cvt<T>::to_f(src[p * K + k]) - m) / sq) / den);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
segment_softmax_bwd_kernel(const T* __restrict__ out, const T* __restrict__ gout,
                           const int64_t* __restrict__ ptr, T* __restrict__ gsrc,
                           int64_t n_seg, int64_t n_items, int64_t K, int scaling) {
  zero_uncovered_rows(gsrc, ptr, n_seg, n_items, K);
  const int64_t total = n_seg * K;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / K, k = t - i * K;
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    if (p1 <= p0) continue;
    float dot = 0.f;
    for (int64_t p = p0; p < p1; ++p)
      dot += Cvt<T>::to_f(out[p * K + k]) * Cvt<T>::to_f(gout[p * K + k]);
    const float inv = scaling ? rsqrtf((float)(p1 - p0)) : 1.f;
    for (int64_t p = p0; p < p1; ++p) {
      const float a = Cvt<T>::to_f(out[p * K + k]);
      gsrc[p * K + k] = Cvt<T>::from_f(a * (Cvt<T>::to_f(gout[p * K + k]) - dot) * inv);
    }
  }
}

// fp32 rows whose width is a multiple of 4 (the [V, G = 4] score rows of every shipped config): a thread owns FOUR
// adjacent columns of a segment and moves them as one 16-byte vector per item -- 4x fewer threads and requests than
// the thread-per-column kernels above, same per-column arithmetic in the same order (results bit-identical).
__global__ void __launch_bounds__(256)
segment_softmax_fwd_v4_kernel(const float* __restrict__ src, const int64_t* __restrict__ ptr, float* __restrict__ out,
                              int64_t n_seg, int64_t n_items, int64_t K, float eps, int scaling) {
  zero_uncovered_rows(out, ptr, n_seg, n_items, K);
  const int64_t K4 = K >> 2, total = n_seg * K4;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / K4, k = (t - i * K4) << 2;
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    if (p1 <= p0) continue;
    const float* s = src + k;
    float4 m = *reinterpret_cast<const float4*>(s + p0 * K);
    for (int64_t p = p0 + 1; p < p1; ++p) {
      const float4 v = *reinterpret_cast<const float4*>(s + p * K);
      m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
    }
    const float sq = scaling ? sqrtf((float)(p1 - p0)) : 1.f;
    float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t p = p0; p < p1; ++p) {
      const float4 v = *reinterpret_cast<const float4*>(s + p * K);
      sum.x += expf((v.x - m.x) / sq); sum.y += expf((v.y - m.y) / sq);
      sum.z += expf((v.z - m.z) / sq); sum.w += expf((v.w - m.w) / sq);
    }
    const float4 den = make_float4(sum.x + eps, sum.y + eps, sum.z + eps, sum.w + eps);
    for (int64_t p = p0; p < p1; ++p) {
      const float4 v = *reinterpret_cast<const float4*>(s + p * K);
      *reinterpret_cast<float4*>(out + p * K + k) =
          make_float4(expf((v.x - m.x) / sq) / den.x, expf((v.y - m.y) / sq) / den.y,
                      expf((v.z - m.z) / sq) / den.z, expf((v.w - m.w) / sq) / den.w);
    }
  }
}

__global__ void __launch_bounds__(256)
segment_softmax_bwd_v4_kernel(const float* __restrict__ out, const float* __restrict__ gout,
                              const int64_t* __restrict__ ptr, float* __restrict__ gsrc, int64_t n_seg,
                              int64_t n_items, int64_t K, int scaling) {
  zero_uncovered_rows(gsrc, ptr, n_seg, n_items, K);
  const int64_t K4 = K >> 2, total = n_seg * K4;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / K4, k = (t - i * K4) << 2;
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    if (p1 <= p0) continue;
    float4 dot = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t p = p0; p < p1; ++p) {
      const float4 a = *reinterpret_cast<const float4*>(out + p * K + k);
      const float4 g = *reinterpret_cast<const float4*>(gout + p * K + k);
      dot.x += a.x * g.x; dot.y += a.y * g.y; dot.z += a.z * g.z; dot.w += a.w * g.w;
    }
    const float inv = scaling ? rsqrtf((float)(p1 - p0)) : 1.f;
    for (int64_t p = p0; p < p1; ++p) {
      const float4 a = *reinterpret_cast<const float4*>(out + p * K + k);
      const float4 g = *reinterpret_cast<const float4*>(gout + p * K + k);
      *reinterpret_cast<float4*>(gsrc + p * K + k) =
          make_float4(a.x * (g.x - dot.x) * inv, a.y * (g.y - dot.y) * inv, a.z * (g.z - dot.z) * inv,
                      a.w * (g.w - dot.w) * inv);
    }
  }
}

// ---- heuristic pool (pooling.py:129-152): arg over one mapping feature, then row pick
__global__ void __launch_bounds__(256)
heuristic_arg_kernel(const float* __restrict__ x_map, int64_t stride, int64_t feat,
                     const int64_t* __restrict__ ptr, int64_t* __restrict__ arg, int64_t N,
                     int64_t V, int use_max) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    int64_t best = V;
    float bv = 0.f;
    for (int64_t p = p0; p < p1; ++p) {
      const float v = x_map[p * stride + feat];
      if (p == p0 || (use_max ? v > bv : v < bv)) { bv = v; best = p; }
    }
    arg[i] = best;
  }
}

template <typename T, int VEC>
__global__ void __launch_bounds__(256)
pick_rows_kernel(const T* __restrict__ x, const int64_t* __restrict__ arg, T* __restrict__ out,
                 int64_t N, int64_t V, int64_t C) {
  const int64_t CV = C / VEC;
  const int64_t total = N * CV;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / CV, cv = t - i * CV;
    const int64_t j = arg[i];
    Pack<T, VEC> o;
    if (j >= 0 && j < V) {
      o = *reinterpret_cast<const Pack<T, VEC>*>(x + j * C + cv * VEC);
    } else {
#pragma unroll
      for (int q = 0; q < VEC; ++q) o.v[q] = Cvt<T>::from_f(0.f);
    }
    *reinterpret_cast<Pack<T, VEC>*>(out + i * C + cv * VEC) = o;
  }
}

// ---- rows scatter-add: dst[idx[v], :] += src[v, :]  (dst fp32, pre-zeroed by the caller) --------------
// backward of a row gather x[idx] with repeated rows (a caller-supplied row_index that is not a
// permutation, pooling.py `x_mod[idx]`), and of HeuristicBimodalCSRPool's row pick (pooling.py:146-150;
// idx[i] == n_rows marks "no view": skipped).  red.global.add.v4.f32: one instruction per four channels.
template <typename T, int VEC>
__global__ void __launch_bounds__(256)
scatter_add_rows_kernel(const T* __restrict__ src, const int64_t* __restrict__ idx, float* __restrict__ dst,
                        int64_t V, int64_t R, int64_t C) {
  const int64_t CV = C / VEC, total = V * CV;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = t / CV, cv = t - v * CV;
    const int64_t r = idx[v];
    if (r < 0 || r >= R) continue;
    float f[VEC];
    if constexpr (VEC == 1) { f[0] = Cvt<T>::to_f(src[v * C + cv]); atomicAdd(dst + r * C + cv, f[0]); }
    else {
      unpack16<T, VEC>(*reinterpret_cast<const uint4*>(src + v * C + cv * VEC), f);
      float* d = dst + r * C + cv * VEC;
#pragma unroll
      for (int j = 0; j < VEC; j += 4) red_add_v4(d + j, f[j], f[j + 1], f[j + 2], f[j + 3]);
    }
  }
}

// ---- deterministic rows scatter-add (torch.use_deterministic_algorithms) ------------------------------
// Same result as above up to the summation order, which is fixed here: the source rows are bucketed by
// destination row (bucket_sort.cuh, stable: ascending v) and the threads of one row's chunks sum them in
// that order, acc = __fadd_rn(acc, src[v]) from +0.0f.  Every row of dst is written (no pre-zeroing).
struct RowKey {
  const int64_t* idx; int64_t R;
  __device__ __forceinline__ void operator()(int64_t v, int64_t (&k)[1]) const {
    const int64_t r = idx[v];
    k[0] = (r < 0 || r >= R) ? -1 : r;
  }
};

template <typename T, int VEC>
__global__ void __launch_bounds__(256)
scatter_add_rows_det_kernel(const T* __restrict__ src, const int64_t* __restrict__ off,
                            const int64_t* __restrict__ sorted, float* __restrict__ dst, int64_t R, int64_t C) {
  const int64_t CV = C / VEC, total = R * CV;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / CV, cv = t - r * CV;
    const int64_t e1 = off[r + 1];
    float acc[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
    for (int64_t e = off[r]; e < e1; ++e) {
      const int64_t v = sorted[e];
      float f[VEC];
      if constexpr (VEC == 1) f[0] = Cvt<T>::to_f(src[v * C + cv]);
      else unpack16<T, VEC>(__ldg(reinterpret_cast<const uint4*>(src + v * C + cv * VEC)), f);
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc[j] = __fadd_rn(acc[j], f[j]);
    }
    if constexpr (VEC == 1) {
      dst[r * C + cv] = acc[0];
    } else {
      float4* o = reinterpret_cast<float4*>(dst + r * C + cv * VEC);
#pragma unroll
      for (int j = 0; j < VEC; j += 4) o[j / 4] = make_float4(acc[j], acc[j + 1], acc[j + 2], acc[j + 3]);
    }
  }
}

// ---- host-side dispatch ---------------------------------------------------------------------
// Grid-stride launches of 256 threads, at most 16 CTAs per SM (2048 threads per SM, twice over).
template <typename T, int VEC>
static int seg_fwd_launch(const void* src, const int64_t* ptr, void* out, int64_t* arg,
                          int64_t n_seg, int64_t n_items, int64_t K, int reduce,
                          cudaStream_t st) {
  const int grid = grid_cap(n_seg * (K / VEC), 256, 16);
  if (!with_reduce(reduce, [&](auto red) {
        segment_csr_fwd_kernel<T, VEC, decltype(red)::value><<<grid, 256, 0, st>>>((const T*)src, ptr, (T*)out, arg,
                                                                                  n_seg, n_items, K);
      }))
    return fail(DVA_EINVAL, "segment_csr_fwd: unknown reduce");
  return check_launch("segment_csr_fwd");
}

template <typename T, int VEC>
static int seg_bwd_launch(const void* gout, const int64_t* ptr, const int64_t* arg, void* gsrc,
                          int64_t n_seg, int64_t n_items, int64_t K, int reduce, cudaStream_t st) {
  const int grid = grid_cap(n_seg * (K / VEC), 256, 16);
  if (!with_reduce(reduce, [&](auto red) {
        segment_csr_bwd_kernel<T, VEC, decltype(red)::value><<<grid, 256, 0, st>>>((const T*)gout, ptr, arg, (T*)gsrc,
                                                                                  n_seg, n_items, K);
      }))
    return fail(DVA_EINVAL, "segment_csr_bwd: unknown reduce");
  return check_launch("segment_csr_bwd");
}

// no segment at all: every element-level output row is uncovered
static int zero_all_rows(void* dst, int64_t n_items, int64_t K, int dtype, cudaStream_t st) {
  if (!dst) return fail(DVA_EINVAL, "null output");
  const size_t es = dtype == DVA_F32 ? 4 : 2;
  const cudaError_t e = cudaMemsetAsync(dst, 0, (size_t)n_items * (size_t)K * es, st);
  return e == cudaSuccess ? DVA_OK : fail((int)e, "memset failed");
}

}  // namespace dva

using namespace dva;

extern "C" int dva_segment_csr_fwd(const void* src, const int64_t* ptr, void* out, int64_t* arg,
                                   int64_t n_seg, int64_t n_items, int64_t K, int reduce,
                                   int dtype, void* stream) {
  if (n_seg < 0 || n_items < 0 || K < 0) return fail(DVA_EINVAL, "segment_csr_fwd: negative size");
  if (n_seg == 0 || K == 0) return DVA_OK;
  if (!src && n_items > 0) return fail(DVA_EINVAL, "segment_csr_fwd: null src");
  if (!ptr || !out) return fail(DVA_EINVAL, "segment_csr_fwd: null ptr/out");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "segment_csr_fwd: unknown dtype");
  cudaStream_t st = (cudaStream_t)stream;
  return with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    if (vec16_ok<T>(K, src, out))
      return seg_fwd_launch<T, Vec16<T>::N>(src, ptr, out, arg, n_seg, n_items, K, reduce, st);
    return seg_fwd_launch<T, 1>(src, ptr, out, arg, n_seg, n_items, K, reduce, st);
  });
}

extern "C" int dva_segment_csr_bwd(const void* grad_out, const int64_t* ptr, const int64_t* arg,
                                   void* grad_src, int64_t n_seg, int64_t n_items, int64_t K,
                                   int reduce, int dtype, void* stream) {
  if (n_seg < 0 || n_items < 0 || K < 0) return fail(DVA_EINVAL, "segment_csr_bwd: negative size");
  if (K == 0 || n_items == 0) return DVA_OK;
  if (n_seg == 0) return zero_all_rows(grad_src, n_items, K, dtype, (cudaStream_t)stream);
  if (!grad_out || !ptr || !grad_src) return fail(DVA_EINVAL, "segment_csr_bwd: null pointer");
  if ((reduce == DVA_MAX || reduce == DVA_MIN) && !arg)
    return fail(DVA_EINVAL, "segment_csr_bwd: max/min need arg");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "segment_csr_bwd: unknown dtype");
  cudaStream_t st = (cudaStream_t)stream;
  return with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    if (vec16_ok<T>(K, grad_out, grad_src))
      return seg_bwd_launch<T, Vec16<T>::N>(grad_out, ptr, arg, grad_src, n_seg, n_items, K, reduce, st);
    return seg_bwd_launch<T, 1>(grad_out, ptr, arg, grad_src, n_seg, n_items, K, reduce, st);
  });
}

extern "C" int dva_gather_csr(const void* src, const int64_t* ptr, void* out, int64_t n_seg,
                              int64_t n_items, int64_t K, int dtype, void* stream) {
  if (n_seg < 0 || n_items < 0 || K < 0) return fail(DVA_EINVAL, "gather_csr: negative size");
  if (K == 0 || n_items == 0) return DVA_OK;
  if (n_seg == 0) return zero_all_rows(out, n_items, K, dtype, (cudaStream_t)stream);
  if (!src || !ptr || !out) return fail(DVA_EINVAL, "gather_csr: null pointer");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "gather_csr: unknown dtype");
  cudaStream_t st = (cudaStream_t)stream;
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    if (vec16_ok<T>(K, src, out)) {
      constexpr int VEC = Vec16<T>::N;
      gather_csr_kernel<T, VEC><<<grid_cap(n_seg * (K / VEC), 256, 16), 256, 0, st>>>(
          (const T*)src, ptr, (T*)out, n_seg, n_items, K);
    } else {
      gather_csr_kernel<T, 1><<<grid_cap(n_seg * K, 256, 16), 256, 0, st>>>((const T*)src, ptr, (T*)out,
                                                                            n_seg, n_items, K);
    }
  });
  return check_launch("gather_csr");
}

extern "C" int dva_segment_softmax_csr_fwd(const void* src, const int64_t* ptr, void* out,
                                           int64_t n_seg, int64_t n_items, int64_t K, float eps,
                                           int scaling, int dtype, void* stream) {
  if (n_seg < 0 || n_items < 0 || K < 0) return fail(DVA_EINVAL, "segment_softmax_fwd: negative size");
  if (K == 0 || n_items == 0) return DVA_OK;
  if (n_seg == 0) return zero_all_rows(out, n_items, K, dtype, (cudaStream_t)stream);
  if (!src || !ptr || !out) return fail(DVA_EINVAL, "segment_softmax_fwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DVA_F32 && vec16_ok<float>(K, src, out)) {
    segment_softmax_fwd_v4_kernel<<<grid_cap(n_seg * (K / 4), 256, 16), 256, 0, st>>>(
        (const float*)src, ptr, (float*)out, n_seg, n_items, K, eps, scaling);
    return check_launch("segment_softmax_fwd");
  }
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "segment_softmax_fwd: unknown dtype");
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    segment_softmax_fwd_kernel<T><<<grid_cap(n_seg * K, 256, 16), 256, 0, st>>>(
        (const T*)src, ptr, (T*)out, n_seg, n_items, K, eps, scaling);
  });
  return check_launch("segment_softmax_fwd");
}

extern "C" int dva_segment_softmax_csr_bwd(const void* out, const void* grad_out,
                                           const int64_t* ptr, void* grad_src, int64_t n_seg,
                                           int64_t n_items, int64_t K, int scaling, int dtype,
                                           void* stream) {
  if (n_seg < 0 || n_items < 0 || K < 0) return fail(DVA_EINVAL, "segment_softmax_bwd: negative size");
  if (K == 0 || n_items == 0) return DVA_OK;
  if (n_seg == 0) return zero_all_rows(grad_src, n_items, K, dtype, (cudaStream_t)stream);
  if (!out || !grad_out || !ptr || !grad_src) return fail(DVA_EINVAL, "segment_softmax_bwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == DVA_F32 && vec16_ok<float>(K, out, grad_out, grad_src)) {
    segment_softmax_bwd_v4_kernel<<<grid_cap(n_seg * (K / 4), 256, 16), 256, 0, st>>>(
        (const float*)out, (const float*)grad_out, ptr, (float*)grad_src, n_seg, n_items, K, scaling);
    return check_launch("segment_softmax_bwd");
  }
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "segment_softmax_bwd: unknown dtype");
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    segment_softmax_bwd_kernel<T><<<grid_cap(n_seg * K, 256, 16), 256, 0, st>>>(
        (const T*)out, (const T*)grad_out, ptr, (T*)grad_src, n_seg, n_items, K, scaling);
  });
  return check_launch("segment_softmax_bwd");
}

extern "C" int dva_heuristic_pool_fwd(const void* x_mod, const float* x_map, int64_t map_stride,
                                      int64_t feat, const int64_t* ptr, void* out, int64_t* arg,
                                      int64_t N, int64_t V, int64_t C, int use_max, int dtype,
                                      void* stream) {
  if (N < 0 || V < 0 || C < 0 || feat < 0 || feat >= map_stride)
    return fail(DVA_EINVAL, "heuristic_pool: bad sizes");
  if (N == 0) return DVA_OK;
  if (!ptr || !out || !arg || (V > 0 && (!x_mod || !x_map)))
    return fail(DVA_EINVAL, "heuristic_pool: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  heuristic_arg_kernel<<<grid_cap(N, 256, 16), 256, 0, st>>>(x_map, map_stride, feat, ptr, arg, N, V, use_max);
  int rc = check_launch("heuristic_arg");
  if (rc) return rc;
  if (C == 0) return DVA_OK;
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "heuristic_pool: unknown dtype");
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    if (vec16_ok<T>(C, x_mod, out)) {
      constexpr int VEC = Vec16<T>::N;
      pick_rows_kernel<T, VEC><<<grid_cap(N * (C / VEC), 256, 16), 256, 0, st>>>((const T*)x_mod, arg, (T*)out, N, V, C);
    } else {
      pick_rows_kernel<T, 1><<<grid_cap(N * C, 256, 16), 256, 0, st>>>((const T*)x_mod, arg, (T*)out, N, V, C);
    }
  });
  return check_launch("pick_rows");
}

extern "C" int dva_scatter_add_rows(const void* src, const int64_t* idx, float* dst, int64_t V, int64_t R,
                                    int64_t C, int dtype, void* stream) {
  if (V < 0 || R < 0 || C < 0) return fail(DVA_EINVAL, "scatter_add_rows: negative size");
  if (V == 0 || C == 0) return DVA_OK;
  if (!src || !idx || !dst) return fail(DVA_EINVAL, "scatter_add_rows: null pointer");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "scatter_add_rows: unknown dtype");
  cudaStream_t st = (cudaStream_t)stream;
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    if (vec16_ok<T>(C, src, dst)) {
      constexpr int VEC = Vec16<T>::N;
      scatter_add_rows_kernel<T, VEC><<<grid_cap(V * (C / VEC), 256, 16), 256, 0, st>>>((const T*)src, idx, dst, V, R, C);
    } else {
      scatter_add_rows_kernel<T, 1><<<grid_cap(V * C, 256, 16), 256, 0, st>>>((const T*)src, idx, dst, V, R, C);
    }
  });
  return check_launch("scatter_add_rows");
}

static size_t scatter_rows_det_carve(uint8_t* base, int64_t V, int64_t R, bk::BucketIndex* w) {
  return bk::carve_index(base, V, R, w);
}

extern "C" size_t dva_scatter_add_rows_det_workspace_bytes(int64_t V, int64_t R) {
  if (V < 0 || R < 0) return 0;
  return scatter_rows_det_carve(nullptr, V, R, nullptr) + 256;
}

extern "C" int dva_scatter_add_rows_det(const void* src, const int64_t* idx, float* dst, int64_t V, int64_t R,
                                        int64_t C, int dtype, void* workspace, size_t workspace_bytes,
                                        void* stream) {
  if (V < 0 || R < 0 || C < 0) return fail(DVA_EINVAL, "scatter_add_rows_det: negative size");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "scatter_add_rows_det: unknown dtype");
  if (R == 0 || C == 0) return DVA_OK;
  if (!dst) return fail(DVA_EINVAL, "scatter_add_rows_det: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (V == 0) {          // nothing scattered: all rows are zero
    const cudaError_t e = cudaMemsetAsync(dst, 0, (size_t)(R * C) * 4, st);
    return e == cudaSuccess ? DVA_OK : fail((int)e, "scatter_add_rows_det: memset failed");
  }
  if (!src || !idx || !workspace) return fail(DVA_EINVAL, "scatter_add_rows_det: null pointer");
  if (workspace_bytes < dva_scatter_add_rows_det_workspace_bytes(V, R))
    return fail(DVA_EINVAL, "scatter_add_rows_det: workspace too small");
  bk::BucketIndex w;
  scatter_rows_det_carve(align256(workspace), V, R, &w);
  int rc = bk::build_index<1>(RowKey{idx, R}, V, R, w, st);
  if (rc) return rc;
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    if (vec16_ok<T>(C, src, dst)) {
      constexpr int VEC = Vec16<T>::N;
      scatter_add_rows_det_kernel<T, VEC><<<grid_cap(R * (C / VEC), 256, 16), 256, 0, st>>>((const T*)src, w.off, w.sorted,
                                                                                            dst, R, C);
    } else {
      scatter_add_rows_det_kernel<T, 1><<<grid_cap(R * C, 256, 16), 256, 0, st>>>((const T*)src, w.off, w.sorted, dst, R, C);
    }
  });
  return check_launch("scatter_add_rows_det");
}
