// Native construction of the two-level point -> view -> pixel CSR (ImageMapping) from an unordered list
// of (point, image, pixel) items, and the re-indexing operations built on it:
//   ImageMapping.from_dense               image.py:1728-1795   (MapImages, every dataset build)
//   ImageMapping.select_points('merge')   image.py:2211-2273   (after every strided 3D conv, modules.py:232)
//   ImageData.view_cat_sorting            image.py:1549-1574   (every forward of a multi-setting branch)
// The reference composes these from lexargsort / lexargunique (composite int64 key -> full sort ->
// unique), scatter_mean, repeat_interleave and cumsum, with several host synchronisations (.item(), max).
//
// Here: items are BUCKETED by point (csrc/bucket_sort.cuh) -- the point id is a dense integer in [0, num_points), so the top
// level of the CSR is a counting sort (histogram + exclusive scan + scatter), not a comparison sort --
// and each point's handful of items is then ordered by one warp with a rank sort on the key
// (image, [x, y,] source index).  Runs of equal image inside a point are its views; their pixels follow
// in order.  Everything is integer, deterministic (the source index breaks every tie, i.e. the result
// equals a STABLE lexicographic sort) and enqueued on the caller's stream; the only value the host needs
// is the pair (V, P) of output sizes, written to a device word the caller reads once.
//
// HBM-bound integer work: per item ~6 passes of 8..24 bytes; no tensor cores.
#include "bucket_sort.cuh"

namespace dva {
namespace mb {

// point id of an item as its bucket key; out-of-range ids set status bit 0 (reported to the host with the
// sizes) and drop the item
struct PointKey {
  const int64_t* point; int64_t num_points; int32_t* status;
  __device__ __forceinline__ void operator()(int64_t i, int64_t (&k)[1]) const {
    const int64_t p = point[i];
    const bool ok = p >= 0 && p < num_points;
    if (!ok && status) atomicOr(status, 1);
    k[0] = ok ? p : -1;
  }
};

template <typename PIX> struct PixIO;
template <> struct PixIO<int16_t> { static __device__ __forceinline__ void ld(const void* p, int64_t i, int& x, int& y) { const short2 v = reinterpret_cast<const short2*>(p)[i]; x = v.x; y = v.y; }
                                    static __device__ __forceinline__ void st(void* p, int64_t i, int x, int y) { reinterpret_cast<short2*>(p)[i] = make_short2((short)x, (short)y); } };
template <> struct PixIO<int32_t> { static __device__ __forceinline__ void ld(const void* p, int64_t i, int& x, int& y) { const int2 v = reinterpret_cast<const int2*>(p)[i]; x = v.x; y = v.y; }
                                    static __device__ __forceinline__ void st(void* p, int64_t i, int x, int y) { reinterpret_cast<int2*>(p)[i] = make_int2(x, y); } };
template <> struct PixIO<int64_t> { static __device__ __forceinline__ void ld(const void* p, int64_t i, int& x, int& y) { const longlong2 v = reinterpret_cast<const longlong2*>(p)[i]; x = (int)v.x; y = (int)v.y; }
                                    static __device__ __forceinline__ void st(void* p, int64_t i, int x, int y) { reinterpret_cast<longlong2*>(p)[i] = make_longlong2(x, y); } };

// key of an item inside its point: (image, [x, y]) then the source index (stability)
using bk::Key;

template <typename PIX>
__device__ __forceinline__ Key make_key(const int64_t* image, const void* pix, int64_t src, bool by_pixel) {
  Key k; k.src = src;
  int64_t a = image[src];
  if (by_pixel) { int x, y; PixIO<PIX>::ld(pix, src, x, y); a = (a << 32) | ((int64_t)(x & 0xffff) << 16) | (int64_t)(y & 0xffff); }
  k.a = a;
  return k;
}

// One warp per point: rank-sort the bucket, then flag view heads / duplicate pixels and count them.
// flags[pos]: bit 0 = first item of a view, bit 1 = kept pixel.  (x, y must fit 16 bits when by_pixel.)
template <typename PIX>
__global__ void __launch_bounds__(256)
order_points(const int64_t* __restrict__ image, const void* __restrict__ pix, const int64_t* __restrict__ off,
             int64_t* __restrict__ bucket, int64_t* __restrict__ sorted, uint8_t* __restrict__ flags,
             int32_t* __restrict__ n_views, int32_t* __restrict__ n_pix, int64_t num_points, int dedupe) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < num_points; p += warps) {
    const int64_t b0 = off[p], L = off[p + 1] - b0;
    if (L == 0) { if (lane == 0) { n_views[p] = 0; n_pix[p] = 0; } continue; }
    // ---- rank sort (stable through the source index) ----
    bk::warp_rank_sort(bucket, sorted, b0, L, lane,
                       [&](int64_t s) { return make_key<PIX>(image, pix, s, dedupe != 0); });
    __syncwarp();
    // ---- flags and counts over the ordered bucket ----
    int nv = 0, np = 0;
    for (int64_t c = 0; c < L; c += 32) {
      const int64_t j = c + lane;
      bool head = false, keep = false;
      if (j < L) {
        const int64_t s = sorted[b0 + j];
        const int64_t m = image[s];
        head = true; keep = true;
        if (j > 0) {
          const int64_t sp = sorted[b0 + j - 1];
          head = image[sp] != m;
          if (dedupe && !head) {
            int x, y, xp, yp;
            PixIO<PIX>::ld(pix, s, x, y); PixIO<PIX>::ld(pix, sp, xp, yp);
            keep = !(x == xp && y == yp);
          }
        }
        flags[b0 + j] = (uint8_t)((head ? 1 : 0) | (keep ? 2 : 0));
      }
      nv += __popc(__ballot_sync(0xffffffffu, head));
      np += __popc(__ballot_sync(0xffffffffu, keep));
    }
    if (lane == 0) { n_views[p] = nv; n_pix[p] = np; }
  }
}

// One warp per point: write images / atomic pointers / pixels / per-view mean features.
template <typename PIX>
__global__ void __launch_bounds__(256)
emit_points(const int64_t* __restrict__ image, const void* __restrict__ pix, const float* __restrict__ feat,
            const int64_t* __restrict__ feat_row, const uint8_t* __restrict__ feat_on, int F,
            const int64_t* __restrict__ off, const int64_t* __restrict__ sorted, const uint8_t* __restrict__ flags,
            const int64_t* __restrict__ view_ptr, const int64_t* __restrict__ pix_ptr, int64_t num_points,
            int64_t* __restrict__ images_out, int64_t* __restrict__ atomic_ptr, void* __restrict__ pix_out,
            float* __restrict__ feat_out, int64_t* __restrict__ order_out) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < num_points; p += warps) {
    const int64_t b0 = off[p], L = off[p + 1] - b0;
    int64_t v_base = view_ptr[p], q_base = pix_ptr[p];
    for (int64_t c = 0; c < L; c += 32) {
      const int64_t j = c + lane;
      const uint8_t f = j < L ? flags[b0 + j] : 0;
      const unsigned heads = __ballot_sync(0xffffffffu, f & 1), keeps = __ballot_sync(0xffffffffu, f & 2);
      const unsigned below = (1u << lane) - 1u;
      const int64_t v = v_base + __popc(heads & below) + ((f & 1) ? 0 : -1);     // view of this item
      const int64_t q = q_base + __popc(keeps & below);                          // kept-pixel slot
      if (j < L) {
        const int64_t s = sorted[b0 + j];
        if (f & 2) {
          int x, y;
          PixIO<PIX>::ld(pix, s, x, y);
          PixIO<PIX>::st(pix_out, q, x, y);
          if (order_out) order_out[q] = s;
        }
        if (f & 1) {
          images_out[v] = image[s];
          atomic_ptr[v] = q;
          if (feat != nullptr) {          // mean over the view's counted items, in order (views are short)
            float acc[16];
            const int Fc = F < 16 ? F : 16;
            for (int k = 0; k < Fc; ++k) acc[k] = 0.f;
            int cnt = 0;
            for (int64_t t = j; t < L; ++t) {
              if (t > j && (flags[b0 + t] & 1)) break;
              const int64_t st = sorted[b0 + t];
              if (feat_on == nullptr || feat_on[st]) {
                const float* row = feat + (feat_row ? feat_row[st] : st) * (int64_t)F;
                for (int k = 0; k < Fc; ++k) acc[k] += row[k];
                ++cnt;
              }
            }
            const float inv = 1.f / (float)(cnt > 0 ? cnt : 1);
            for (int k = 0; k < Fc; ++k) feat_out[v * (int64_t)F + k] = acc[k] * inv;
          }
        }
      }
      v_base += __popc(heads);
      q_base += __popc(keeps);
    }
  }
}

__global__ void finish_counts(const int64_t* __restrict__ view_ptr, const int64_t* __restrict__ pix_ptr,
                              int64_t num_points, int64_t* __restrict__ atomic_ptr, int64_t* __restrict__ counts,
                              const int32_t* __restrict__ status) {
  const int64_t V = view_ptr[num_points], P = pix_ptr[num_points];
  atomic_ptr[V] = P;
  counts[0] = V; counts[1] = P; counts[2] = *status;
}

// ---- view_cat_sorting (image.py:1549-1574) in closed form ------------------------------------------------
// Settings s = 0..S-1 each hold a view CSR over the same N points.  The permutation that interleaves the
// concatenated views into point order (a stable argsort of the dense point ids) needs no sort:
//   dest(s, p, j) = sum_s' ptr_s'[p] + sum_{s' < s} (ptr_s'[p+1] - ptr_s'[p]) + (j - ptr_s[p]);  sorting[dest] = base_s + j
__global__ void __launch_bounds__(256)
view_cat_sorting_kernel(const int64_t* const* __restrict__ ptrs, const int64_t* __restrict__ bases, int S,
                        int64_t N, int64_t* __restrict__ sorting, int64_t* __restrict__ csr_cat) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p <= N; p += (int64_t)gridDim.x * blockDim.x) {
    int64_t start = 0;
    for (int s = 0; s < S; ++s) start += ptrs[s][p];
    csr_cat[p] = start;
    if (p == N) continue;
    int64_t d = start;
    for (int s = 0; s < S; ++s) {
      const int64_t a = ptrs[s][p], b = ptrs[s][p + 1];
      for (int64_t j = a; j < b; ++j) sorting[d++] = bases[s] + j;
    }
  }
}

struct Workspace {
  int32_t *cnt, *cursor, *n_views, *n_pix, *status;
  int64_t *off, *pix_ptr, *bucket, *sorted, *block_sums;
  uint8_t* flags;
};

static size_t carve(uint8_t* base, int64_t n, int64_t N, Workspace* w) {
  size_t o = 0;
  auto take = [&](size_t bytes) { uint8_t* p = base ? base + o : nullptr; o += round256(bytes); return p; };
  const int64_t nb = bk::scan_block_words(N);
  uint8_t* p;
  p = take((size_t)(N + 1) * 4); if (w) w->cnt = (int32_t*)p;
  p = take((size_t)(N + 1) * 4); if (w) w->cursor = (int32_t*)p;
  p = take((size_t)(N + 1) * 4); if (w) w->n_views = (int32_t*)p;
  p = take((size_t)(N + 1) * 4); if (w) w->n_pix = (int32_t*)p;
  p = take(256); if (w) w->status = (int32_t*)p;
  p = take((size_t)(N + 1) * 8); if (w) w->off = (int64_t*)p;
  p = take((size_t)(N + 1) * 8); if (w) w->pix_ptr = (int64_t*)p;
  p = take((size_t)(n + 1) * 8); if (w) w->bucket = (int64_t*)p;
  p = take((size_t)(n + 1) * 8); if (w) w->sorted = (int64_t*)p;
  p = take((size_t)nb * 8); if (w) w->block_sums = (int64_t*)p;
  p = take((size_t)(n + 1)); if (w) w->flags = p;
  return o;
}

}  // namespace mb
}  // namespace dva

using namespace dva;

extern "C" size_t dva_mapping_build_workspace_bytes(int64_t n_items, int64_t num_points) {
  if (n_items < 0 || num_points < 0) return 0;
  return mb::carve(nullptr, n_items, num_points, nullptr) + 256;
}

// See include/dva_b200.h.  pix_code: 0 = int16, 1 = int32, 2 = int64 pairs (x, y).
extern "C" int dva_mapping_build(const int64_t* point_ids, const int64_t* image_ids, const void* pixels, int pix_code,
                                 const float* feat, const int64_t* feat_row, const uint8_t* feat_on, int64_t F,
                                 int64_t n_items, int64_t num_points, int dedupe_pixels, int64_t* view_ptr,
                                 int64_t* images_out, int64_t* atomic_ptr, void* pixels_out, float* feat_out,
                                 int64_t* order_out, int64_t* counts, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  if (n_items < 0 || num_points < 0 || F < 0 || F > 16 || pix_code < 0 || pix_code > 2)
    return fail(DVA_EINVAL, "mapping_build: bad sizes (F <= 16, pix_code in 0..2)");
  if (n_items >= (1ll << 31)) return fail(DVA_EUNSUPPORTED, "mapping_build: more than 2^31 items");
  if (!view_ptr || !counts || !atomic_ptr || !workspace) return fail(DVA_EINVAL, "mapping_build: null pointer");
  if (n_items > 0 && (!point_ids || !image_ids || !pixels || !images_out || !pixels_out || (feat && !feat_out)))
    return fail(DVA_EINVAL, "mapping_build: null pointer");
  if (workspace_bytes < dva_mapping_build_workspace_bytes(n_items, num_points)) return fail(DVA_EINVAL, "mapping_build: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  mb::Workspace w;
  mb::carve(align256(workspace), n_items, num_points, &w);
  cudaError_t e = cudaMemsetAsync(w.cnt, 0, (size_t)((uint8_t*)w.n_views - (uint8_t*)w.cnt), st);   // cnt + cursor
  if (e == cudaSuccess) e = cudaMemsetAsync(w.status, 0, 256, st);
  if (e != cudaSuccess) return fail((int)e, "mapping_build: memset failed");
  int rc;
  if (n_items > 0) {
    bk::count_keys<1><<<grid_cap(n_items, 256, 16), 256, 0, st>>>(mb::PointKey{point_ids, num_points, w.status}, n_items,
                                                             num_points, w.cnt);
    if ((rc = check_launch("mb_count_points"))) return rc;
  }
  if ((rc = bk::exclusive_scan(w.cnt, num_points, w.off, w.block_sums, st))) return rc;
  if (n_items > 0) {
    bk::scatter_keys<1><<<grid_cap(n_items, 256, 16), 256, 0, st>>>(mb::PointKey{point_ids, num_points, nullptr}, n_items,
                                                               num_points, w.off, w.cursor, w.bucket);
    if ((rc = check_launch("mb_scatter_items"))) return rc;
  }
  const int pgrid = grid_cap(num_points * 32, 256, 16);
  if (num_points > 0) {
    with_pix(pix_code, [&](auto p) {
      mb::order_points<decltype(p)><<<pgrid, 256, 0, st>>>(image_ids, pixels, w.off, w.bucket, w.sorted, w.flags, w.n_views,
                                                           w.n_pix, num_points, dedupe_pixels);
    });
    if ((rc = check_launch("mb_order_points"))) return rc;
  }
  if ((rc = bk::exclusive_scan(w.n_views, num_points, view_ptr, w.block_sums, st))) return rc;
  if ((rc = bk::exclusive_scan(w.n_pix, num_points, w.pix_ptr, w.block_sums, st))) return rc;
  if (num_points > 0 && n_items > 0) {
    with_pix(pix_code, [&](auto p) {
      mb::emit_points<decltype(p)><<<pgrid, 256, 0, st>>>(image_ids, pixels, feat, feat_row, feat_on, (int)F, w.off,
                                                          w.sorted, w.flags, view_ptr, w.pix_ptr, num_points, images_out,
                                                          atomic_ptr, pixels_out, feat_out, order_out);
    });
    if ((rc = check_launch("mb_emit_points"))) return rc;
  }
  mb::finish_counts<<<1, 1, 0, st>>>(view_ptr, w.pix_ptr, num_points, atomic_ptr, counts, w.status);
  return check_launch("mb_finish_counts");
}

// sorting [V_total] and csr_cat [N + 1] of S settings whose view pointers (device arrays [N + 1]) are listed in
// ptrs (device array of S device pointers); bases[s] = number of views of the settings before s.
extern "C" int dva_view_cat_sorting(const int64_t* const* ptrs, const int64_t* bases, int64_t S, int64_t N,
                                    int64_t* sorting, int64_t* csr_cat, void* stream) {
  if (S < 1 || N < 0) return fail(DVA_EINVAL, "view_cat_sorting: bad sizes");
  if (!ptrs || !bases || !csr_cat) return fail(DVA_EINVAL, "view_cat_sorting: null pointer");
  mb::view_cat_sorting_kernel<<<grid_cap(N + 1, 256, 16), 256, 0, (cudaStream_t)stream>>>(ptrs, bases, (int)S, N, sorting, csr_cat);
  return check_launch("view_cat_sorting");
}
