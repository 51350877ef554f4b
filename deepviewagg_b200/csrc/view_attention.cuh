// Shared between the three implementations of the fused view-attention pair:
//   view_attention.cu       streaming kernels, forward and backward (row chunks live in registers; best for
//                           long segments of >= 512-byte rows); host dispatch and the C ABI
//   view_attention_ring.cu  ring kernels, forward and backward (rows staged in shared memory by cp.async /
//                           bulk copies, several batches in flight per warp across point boundaries; best for
//                           short segments and rows <= 512 bytes)
//   view_attention_lane.cu  lane-per-view backward (a warp takes a group of points holding <= 32 views; rows
//                           by bulk copy, one per view lane)
// The per-point arithmetic below is written once for all of them; the attention weight itself is not, each
// kernel keeps its own exp / division form.
#pragma once
#include "dva_common.cuh"

namespace dva {

struct VAParams {
  const void* x; const void* idx; int idx64;
  const float* compat; const int64_t* ptr;
  const float* gate_w; const float* gate_b;
  // fwd
  void* out; float* att; float* seg_max; float* seg_den; int32_t* seg_arg;
  // bwd
  const void* gout; const float* s_max; const float* s_den; const int32_t* s_arg;
  void* gx; float* gcompat; float* gate_partial; int scatter;
  int64_t N, V, R;
  int C, G, group_scaling;
  float eps;
};

constexpr int kTileStride = 33;    // att tile is [G][33]: (g,v) -> bank (g+v)%32, conflict-free

// reduce over the lanes that share (lane % G): offsets 16 .. G
__device__ __forceinline__ float group_lane_sum(float v, int G) {
  for (int off = 16; off >= G; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// ---- shared memory, mbarrier and bulk async copy (ring and lane kernels)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
// makes the initialised barriers visible to the async proxy
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  }
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// x row of view v (identity when there is no index; the host guarantees R < 2^32)
__device__ __forceinline__ uint32_t load_row_id(const void* idx, int idx64, int64_t v) {
  if (idx == nullptr) return (uint32_t)v;
  return idx64 ? (uint32_t) reinterpret_cast<const int64_t*>(idx)[v]
               : (uint32_t) reinterpret_cast<const int32_t*>(idx)[v];
}
__device__ __forceinline__ float sel4(const float4& v, int g) {
  return g == 0 ? v.x : (g == 1 ? v.y : (g == 2 ? v.z : v.w));
}

// ---- per-point math of one group g (gradients: see view_attention.cu)
// gate on the group's max score m: z = w m + b, t = tanh(relu(z))
__device__ __forceinline__ float gate_t(float z) { return tanhf(fmaxf(z, 0.f)); }
__device__ __forceinline__ float4 gate_z4(const float4& w, const float4& m, const float4& b) {
  return make_float4(fmaf(w.x, m.x, b.x), fmaf(w.y, m.y, b.y), fmaf(w.z, m.z, b.z), fmaf(w.w, m.w, b.w));
}
__device__ __forceinline__ float4 gate_t4(const float4& z) {
  return make_float4(gate_t(z.x), gate_t(z.y), gate_t(z.z), gate_t(z.w));
}

// Gate gradient with S = sum_v a s' (= t dL/dt): 0 while the gate is closed (z <= 0); otherwise
// u = dL/dt (1 - t^2) and the returned dq = u w flows to the arg-max view's score.  The lanes that `keep` the
// term also accumulate dw += u m, db += u (lanes holding a copy of the same point's term pass false).
__device__ __forceinline__ float gate_grad(float S, float z, float t, float w, float m, bool keep, float& dw,
                                           float& db) {
  if (!(z > 0.f)) return 0.f;
  const float dLdt = (t != 0.f) ? S / t : 0.f;
  const float u = dLdt * (1.f - t * t);
  const float dq = u * w;
  if (keep) {
    dw += u * m;
    db += u;
  }
  return dq;
}
__device__ __forceinline__ float4 gate_grad4(const float4& S, const float4& z, const float4& t, const float4& w,
                                             const float4& m, bool keep, float4& dw, float4& db) {
  return make_float4(gate_grad(S.x, z.x, t.x, w.x, m.x, keep, dw.x, db.x),
                     gate_grad(S.y, z.y, t.y, w.y, m.y, keep, dw.y, db.y),
                     gate_grad(S.z, z.z, t.z, w.z, m.z, keep, dw.z, db.z),
                     gate_grad(S.w, z.w, t.w, w.w, m.w, keep, dw.w, db.w));
}

// grad_compat of one view: a (s' - S) / sqrt(n) + [view == arg-max] dq
__device__ __forceinline__ float compat_grad(float a, float sv, float S, float inv_sq, bool is_arg, float dq) {
  float d = a * (sv - S) * inv_sq;
  if (is_arg) d += dq;
  return d;
}
__device__ __forceinline__ float4 compat_grad4(const float4& a, const float4& sv, const float4& S, float inv_sq,
                                               int v, const int4& arg, const float4& dq) {
  return make_float4(compat_grad(a.x, sv.x, S.x, inv_sq, v == arg.x, dq.x),
                     compat_grad(a.y, sv.y, S.y, inv_sq, v == arg.y, dq.y),
                     compat_grad(a.z, sv.z, S.z, inv_sq, v == arg.z, dq.z),
                     compat_grad(a.w, sv.w, S.w, inv_sq, v == arg.w, dq.w));
}

// Gate parameter gradients of a G = 4 backward CTA of WARPS warps: lane partials -> warp -> block partial
// (fixed order, deterministic) -> partial[blockIdx.x][dw0..3, db0..3].  Every thread of the CTA calls it.
template <int WARPS>
__device__ __forceinline__ void store_gate_partial(float* __restrict__ partial, const float4& dw, const float4& db) {
  __shared__ float gate_s[WARPS][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float v[8] = {dw.x, dw.y, dw.z, dw.w, db.x, db.y, db.z, db.w};
#pragma unroll
  for (int q = 0; q < 8; ++q) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < 8; ++q) gate_s[warp][q] = v[q];
  }
  __syncthreads();
  if ((int)threadIdx.x < 8) {
    float acc = 0.f;
    for (int w = 0; w < WARPS; ++w) acc += gate_s[w][threadIdx.x];
    partial[(int64_t)blockIdx.x * 8 + threadIdx.x] = acc;
  }
}

// ---- host side
// Persistent grid of the ring and lane kernels, whose warps take ranges of points: the co-resident CTAs (kNumSMs x
// occupancy, at most max_ctas_per_sm per SM) ...
template <typename K>
int resident_ctas(K kern, size_t smem, int warps_per_cta, int max_ctas_per_sm, const char* what, int64_t* ctas_out) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return failf((int)e, "%s: %zu bytes of shared memory: %s", what, smem, cudaGetErrorString(e));
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, warps_per_cta * 32, smem) != cudaSuccess || occ < 1) occ = 1;
  if (occ > max_ctas_per_sm) occ = max_ctas_per_sm;
  *ctas_out = (int64_t)kNumSMs * occ;
  return DVA_OK;
}
// ... and no more CTAs than it takes to give every warp one of n_ranges
inline int range_grid(int64_t ctas, int warps_per_cta, int64_t n_ranges) {
  const int64_t need = (n_ranges + warps_per_cta - 1) / warps_per_cta;
  return (int)(ctas > need ? (need < 1 ? 1 : need) : ctas);
}

// The ring kernels' warps stride over ranges of PR points: about ranges_per_warp ranges per warp of the full grid,
// and never fewer than 8 points per range.
template <typename K>
int range_geometry(K kern, size_t smem, int warps_per_cta, int max_ctas_per_sm, int ranges_per_warp, int64_t N,
                   const char* what, int* grid_out, int* pr_out) {
  int64_t ctas = 0;
  if (int rc = resident_ctas(kern, smem, warps_per_cta, max_ctas_per_sm, what, &ctas)) return rc;
  const int64_t slots = ctas * warps_per_cta * ranges_per_warp;
  int64_t pr = (N + slots - 1) / slots;
  if (pr < 8) pr = 8;
  *grid_out = range_grid(ctas, warps_per_cta, (N + pr - 1) / pr); *pr_out = (int)pr;
  return DVA_OK;
}

// The lane backward's warps take ranges of PR points from a queue (a counter the launcher zeroes on the stream):
// ranges of about kLaneRangeViews views -- 8 groups of 32 views, a short wait at the end of the kernel -- but never
// more than kLaneMaxRangePoints points, so that with few views per point the points are still spread over many
// warps; and at most kLaneMaxRanges ranges, which wins over both.  Its gate-gradient partials are one per range,
// [2G = 8][n_ranges], so that they do not depend on which warp took which range.
constexpr int64_t kLaneRangeViews = 256;
constexpr int64_t kLaneMaxRangePoints = 8192;
constexpr int64_t kLaneMaxRanges = 1 << 17;
inline int64_t lane_range_points(int64_t N, int64_t V) {
  int64_t pr = (kLaneRangeViews * N + V - 1) / (V > 0 ? V : 1);
  if (pr > kLaneMaxRangePoints) pr = kLaneMaxRangePoints;
  const int64_t fit = (N + kLaneMaxRanges - 1) / kLaneMaxRanges;   // the workspace holds kLaneMaxRanges partials
  if (pr < fit) pr = fit;
  return pr < 1 ? 1 : pr;
}

// ring kernels (view_attention_ring.cu) and lane-per-view backward (view_attention_lane.cu); the launchers return a
// DVA_* / cudaError code like every other entry point.  Shape / alignment conditions: view_attention.cu.
int va_ring_fwd(const VAParams& P, int dtype, cudaStream_t st);
int va_ring_bwd(const VAParams& P, int dtype, int* grid_out, cudaStream_t st);
// next_range: a counter on the device, zeroed here before the launch
int va_lane_bwd(const VAParams& P, int dtype, int64_t pr, uint32_t* next_range, cudaStream_t st);

}  // namespace dva
