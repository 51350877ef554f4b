// Ragged per-group query.key compatibilities (QKVBimodalCSRPool, pooling.py:499-512).
// The reference expands the per-point queries to views with repeat_interleave (pooling.py:500)
// and reduces a [V,G,D] product; here one thread owns one (point, g*D+d) column, keeps the
// query element in a register and walks the point's views, so Q is read once per point and
// the [V,G*D] expansion never exists.  fp32 throughout (scores feed the softmax statistics).
//   bytes fwd: V*(G*D*4 + G*4) + N*(G*D*4 + 8);  bwd adds V*G*D*4 + N*G*D*4 writes.
#include "dva_common.cuh"

namespace dva {

// fwd: one thread per (point, group); D-loop inside (D is 8 in all shipped configs)
__global__ void __launch_bounds__(256)
qk_scores_fwd_kernel(const float* __restrict__ keys, const float* __restrict__ queries,
                     const int64_t* __restrict__ ptr, float* __restrict__ compat, int64_t N,
                     int G, int D, float scale) {
  const int64_t total = N * G;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / G;
    const int g = (int)(t - i * G);
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    const float* q = queries + i * (int64_t)G * D + g * D;
    for (int64_t v = p0; v < p1; ++v) {
      const float* k = keys + v * (int64_t)G * D + g * D;
      float acc = 0.f;
      for (int d = 0; d < D; ++d) acc += k[d] * __ldg(q + d);   // reference order: sum over d
      compat[v * G + g] = acc * scale;
    }
  }
}

// bwd: one thread per (point, g*D+d)
__global__ void __launch_bounds__(256)
qk_scores_bwd_kernel(const float* __restrict__ keys, const float* __restrict__ queries,
                     const int64_t* __restrict__ ptr, const float* __restrict__ gcompat,
                     float* __restrict__ gkeys, float* __restrict__ gqueries, int64_t N, int G,
                     int D, float scale) {
  const int GD = G * D;
  const int64_t total = N * GD;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / GD;
    const int j = (int)(t - i * GD);
    const int g = j / D;
    const int64_t p0 = ptr[i], p1 = ptr[i + 1];
    const float q = queries[i * GD + j];
    float gq = 0.f;
    for (int64_t v = p0; v < p1; ++v) {
      const float gc = gcompat[v * G + g] * scale;
      gkeys[v * GD + j] = gc * q;
      gq = fmaf(gc, keys[v * GD + j], gq);
    }
    gqueries[i * GD + j] = gq;
  }
}

// ---------------------------------------------------------------------------------------------
// vector path (D % 4 == 0, G*D/4 a power of two <= 32; the shipped G = 4, D = 8 gives 8 chunks):
// CPR lanes own the 16-byte chunks of one key row, so a warp serves 32/CPR points at once; the
// query chunk stays in registers for the whole point, a view costs one LDG.128 per lane, and the
// D-sum is a butterfly over the D/4 lanes of a group.  Four views per point are in flight.
// ---------------------------------------------------------------------------------------------
template <int CPR>
__global__ void __launch_bounds__(256)
qk_scores_fwd_vec_kernel(const float4* __restrict__ keys, const float4* __restrict__ queries,
                         const int64_t* __restrict__ ptr, float* __restrict__ compat, int64_t N,
                         int G, int DL /* chunks per group = D/4 */, float scale) {
  constexpr int PPW = 32 / CPR, U = 4;
  const int lane = threadIdx.x & 31, sg = lane / CPR, ck = lane % CPR;
  const int g = ck / DL;
  const bool writer = (ck % DL) == 0;
  const int64_t gwarp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i0 = gwarp * PPW; i0 < N; i0 += nwarps * PPW) {
    const int64_t i = i0 + sg;
    const bool act = i < N;
    const int64_t p0 = act ? ptr[i] : 0;
    const int n = act ? (int)(ptr[i + 1] - p0) : 0;
    const float4 q = act ? __ldg(queries + i * CPR + ck) : make_float4(0.f, 0.f, 0.f, 0.f);
    // the sub-groups of a warp run the same number of steps (shuffles below are warp-wide)
    int nmax = n;
#pragma unroll
    for (int o = CPR; o < 32; o <<= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    for (int v0 = 0; v0 < nmax; v0 += U) {
      float4 k[U];
#pragma unroll
      for (int u = 0; u < U; ++u)
        k[u] = (v0 + u < n) ? __ldg(keys + (p0 + v0 + u) * CPR + ck) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        // reference order within a chunk: sum over d ascending
        float acc = k[u].x * q.x;
        acc = fmaf(k[u].y, q.y, acc); acc = fmaf(k[u].z, q.z, acc); acc = fmaf(k[u].w, q.w, acc);
        for (int o = 1; o < DL; o <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (writer && v0 + u < n) compat[(p0 + v0 + u) * G + g] = acc * scale;
      }
    }
  }
}

template <int CPR>
__global__ void __launch_bounds__(256)
qk_scores_bwd_vec_kernel(const float4* __restrict__ keys, const float4* __restrict__ queries,
                         const int64_t* __restrict__ ptr, const float* __restrict__ gcompat,
                         float4* __restrict__ gkeys, float4* __restrict__ gqueries, int64_t N, int G,
                         int DL, float scale) {
  constexpr int PPW = 32 / CPR, U = 4;
  const int lane = threadIdx.x & 31, sg = lane / CPR, ck = lane % CPR;
  const int g = ck / DL;
  const int64_t gwarp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i0 = gwarp * PPW; i0 < N; i0 += nwarps * PPW) {
    const int64_t i = i0 + sg;
    if (i >= N) continue;
    const int64_t p0 = ptr[i];
    const int n = (int)(ptr[i + 1] - p0);
    const float4 q = __ldg(queries + i * CPR + ck);
    float4 gq = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int v0 = 0; v0 < n; v0 += U) {
      float4 k[U]; float gc[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool ok = v0 + u < n;
        k[u] = ok ? __ldg(keys + (p0 + v0 + u) * CPR + ck) : make_float4(0.f, 0.f, 0.f, 0.f);
        gc[u] = ok ? __ldg(gcompat + (p0 + v0 + u) * G + g) * scale : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (v0 + u < n)
          gkeys[(p0 + v0 + u) * CPR + ck] = make_float4(gc[u] * q.x, gc[u] * q.y, gc[u] * q.z, gc[u] * q.w);
        gq.x = fmaf(gc[u], k[u].x, gq.x); gq.y = fmaf(gc[u], k[u].y, gq.y);
        gq.z = fmaf(gc[u], k[u].z, gq.z); gq.w = fmaf(gc[u], k[u].w, gq.w);
      }
    }
    gqueries[i * CPR + ck] = gq;
  }
}

// CPR for the vector path, or 0
static inline int qk_vec_cpr(int64_t G, int64_t D, const void* a, const void* b, const void* c, const void* d) {
  if (D % 4 != 0) return 0;
  const int64_t cpr = G * D / 4, dl = D / 4;
  if (cpr > 32 || (cpr & (cpr - 1)) != 0 || (dl & (dl - 1)) != 0) return 0;
  if (!aligned16(a) || !aligned16(b) || (c && !aligned16(c)) || (d && !aligned16(d))) return 0;
  return (int)cpr;
}

}  // namespace dva

using namespace dva;

extern "C" int dva_qk_scores_fwd(const float* keys, const float* queries, const int64_t* ptr,
                                 float* compat, int64_t N, int64_t V, int64_t G, int64_t D,
                                 float scale, void* stream) {
  if (N < 0 || V < 0 || G < 1 || D < 1) return fail(DVA_EINVAL, "qk_scores_fwd: bad sizes");
  if (N == 0 || V == 0) return DVA_OK;
  if (!keys || !queries || !ptr || !compat) return fail(DVA_EINVAL, "qk_scores_fwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (const int cpr = qk_vec_cpr(G, D, keys, queries, nullptr, nullptr)) {
    const int grid = grid_cap(N, 8 * (32 / cpr), 16);   // 8 warps of 32 / cpr points
    with_value<1, 2, 4, 8, 16, 32>(cpr, [&](auto c) {
      qk_scores_fwd_vec_kernel<decltype(c)::value><<<grid, 256, 0, st>>>(
          reinterpret_cast<const float4*>(keys), reinterpret_cast<const float4*>(queries), ptr, compat, N, (int)G,
          (int)(D / 4), scale);
    });
    return check_launch("qk_scores_fwd(vec)");
  }
  qk_scores_fwd_kernel<<<grid_cap(N * G, 256, 16), 256, 0, st>>>(keys, queries, ptr, compat, N, (int)G, (int)D, scale);
  return check_launch("qk_scores_fwd");
}

extern "C" int dva_qk_scores_bwd(const float* keys, const float* queries, const int64_t* ptr,
                                 const float* grad_compat, float* grad_keys, float* grad_queries,
                                 int64_t N, int64_t V, int64_t G, int64_t D, float scale,
                                 void* stream) {
  if (N < 0 || V < 0 || G < 1 || D < 1) return fail(DVA_EINVAL, "qk_scores_bwd: bad sizes");
  if (N == 0) return DVA_OK;
  if (!queries || !ptr || !grad_queries || (V > 0 && (!keys || !grad_compat || !grad_keys)))
    return fail(DVA_EINVAL, "qk_scores_bwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (const int cpr = (V > 0) ? qk_vec_cpr(G, D, keys, queries, grad_keys, grad_queries) : 0) {
    const int grid = grid_cap(N, 8 * (32 / cpr), 16);
    with_value<1, 2, 4, 8, 16, 32>(cpr, [&](auto c) {
      qk_scores_bwd_vec_kernel<decltype(c)::value><<<grid, 256, 0, st>>>(
          reinterpret_cast<const float4*>(keys), reinterpret_cast<const float4*>(queries), ptr, grad_compat,
          reinterpret_cast<float4*>(grad_keys), reinterpret_cast<float4*>(grad_queries), N, (int)G, (int)(D / 4), scale);
    });
    return check_launch("qk_scores_bwd(vec)");
  }
  qk_scores_bwd_kernel<<<grid_cap(N * G * D, 256, 16), 256, 0, st>>>(
      keys, queries, ptr, grad_compat, grad_keys, grad_queries, N, (int)G, (int)D, scale);
  return check_launch("qk_scores_bwd");
}
