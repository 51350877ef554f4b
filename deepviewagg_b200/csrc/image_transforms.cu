// Per-sample image transforms on GPU mappings (core/multimodal/transforms.py), integer and bit-exact:
//
//   dva_mapping_image_stats   one pass over views / pixels -> per-image pixel count, bbox, and the
//                             256-bin occupancy of the quantised width (CenterRoll, image.py:1005)
//   dva_center_roll           CenterRoll cost over the candidate rolls, one warp per image
//   dva_image_remap           roll / crop / flip of [B,C,H,W] maps in one copy (NCHW or channels-last)
//   dva_coverage_index/_pick  unseen-point bookkeeping of PickImagesFromMemoryCredit (image.py:804-867)
//
// All accumulations are integer (min / max / add / or / exch / sub), so results do not depend on the
// launch configuration or on the order in which atomics land.
#include "bucket_sort.cuh"

namespace dva {

// ---- (a) per-image statistics ----------------------------------------------------------------------------
// stats layout: count int64 [n]; bbox int32 [n, 4] = (x_min, x_max, y_min, y_max); occ uint32 [n, 8]
static __global__ void __launch_bounds__(256)
stats_init(int64_t* __restrict__ count, int32_t* __restrict__ bbox, uint32_t* __restrict__ occ, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    count[i] = 0;
    bbox[4 * i + 0] = INT32_MAX; bbox[4 * i + 1] = INT32_MIN;
    bbox[4 * i + 2] = INT32_MAX; bbox[4 * i + 3] = INT32_MIN;
    if (occ) for (int k = 0; k < 8; ++k) occ[8 * i + k] = 0u;
  }
}

template <typename PIX>
static __global__ void __launch_bounds__(256)
stats_accumulate(const int64_t* __restrict__ images, const int64_t* __restrict__ aptr, const PIX* __restrict__ pix,
                 int64_t V, int64_t n, float ref_w, int64_t* __restrict__ count, int32_t* __restrict__ bbox,
                 uint32_t* __restrict__ occ) {
  // one thread per view; the lanes of a warp that share an image reduce together (__match_any_sync) and one
  // of them issues the global atomics.  Every lane runs the same number of rounds so the warp stays converged.
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~(int64_t)31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = warp0; base < V; base += stride) {
    const int64_t v = base + lane;
    int64_t img = -1;
    int32_t cnt = 0, xmn = INT32_MAX, xmx = INT32_MIN, ymn = INT32_MAX, ymx = INT32_MIN;
    uint32_t bits[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    if (v < V) {
      img = images[v];
      const int64_t p0 = aptr[v], p1 = aptr[v + 1];
      for (int64_t p = p0; p < p1; ++p) {
        const int32_t x = (int32_t)pix[2 * p], y = (int32_t)pix[2 * p + 1];
        xmn = min(xmn, x); xmx = max(xmx, x); ymn = min(ymn, y); ymx = max(ymx, y);
        if (occ) {
          // (long)(x.float() * 256 / ref_W) in fp32, image.py:1005; .byte() keeps the low 8 bits
          const int q = (int)(int64_t)__fdiv_rn(__fmul_rn((float)x, 256.f), ref_w) & 255;
          bits[q >> 5] |= 1u << (q & 31);
        }
      }
      cnt = (int32_t)(p1 - p0);
      if (cnt == 0 || img < 0 || img >= n) img = -1;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, img);
    const int leader = __ffs(peers) - 1;
    const int32_t s_cnt = (int32_t)__reduce_add_sync(peers, (unsigned)cnt);
    const int32_t s_xmn = __reduce_min_sync(peers, xmn), s_xmx = __reduce_max_sync(peers, xmx);
    const int32_t s_ymn = __reduce_min_sync(peers, ymn), s_ymx = __reduce_max_sync(peers, ymx);
    uint32_t s_bits[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s_bits[k] = occ ? __reduce_or_sync(peers, bits[k]) : 0u;
    if (lane == leader && img >= 0) {
      atomicAdd((unsigned long long*)(count + img), (unsigned long long)s_cnt);
      atomicMin(bbox + 4 * img + 0, s_xmn); atomicMax(bbox + 4 * img + 1, s_xmx);
      atomicMin(bbox + 4 * img + 2, s_ymn); atomicMax(bbox + 4 * img + 3, s_ymx);
      if (occ) {
#pragma unroll
        for (int k = 0; k < 8; ++k) if (s_bits[k]) atomicOr(occ + 8 * img + k, s_bits[k]);
      }
    }
  }
}

// images without pixels: bbox 0 (torch_scatter's empty -> 0)
static __global__ void __launch_bounds__(256)
stats_finalize(const int64_t* __restrict__ count, int32_t* __restrict__ bbox, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (count[i] == 0) for (int k = 0; k < 4; ++k) bbox[4 * i + k] = 0;
}

// ---- (b) CenterRoll ----------------------------------------------------------------------------------------
// one warp per image; lane l owns bins 8l .. 8l+7.  For every candidate roll r (bytes r = 0, step, 2 step, ..
// < 256): w = (b + r) & 255 over the occupied bins b, cost = (w_max - w_min) + int(|(w_max + w_min) / 2 - 128|)
// (image.py:1010-1024, fp32); the first roll of least cost wins; rolling = long(fp32(r / 256) * ref_W).
static __global__ void __launch_bounds__(256)
center_roll_kernel(const uint32_t* __restrict__ occ, int64_t n, int step, float ref_w, int64_t* __restrict__ rollings) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t img = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; img < n; img += warps) {
    const uint32_t word = occ[8 * img + (lane >> 2)];
    const uint32_t mine = (word >> ((lane & 3) * 8)) & 0xffu;        // bins 8 lane + k, k = 0..7
    int best_cost = INT32_MAX, best_r = 0;
    for (int r = 0; r < 256; r += step) {
      int mn = 256, mx = -1;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (mine & (1u << k)) {
          const int w = (8 * lane + k + r) & 255;
          mn = min(mn, w); mx = max(mx, w);
        }
      mn = __reduce_min_sync(0xffffffffu, mn);
      mx = __reduce_max_sync(0xffffffffu, mx);
      if (mx < 0) { mn = 0; mx = 0; }                                 // no bins: scatter's empty -> 0
      const float c = __fsub_rn(__fdiv_rn(__fadd_rn((float)mx, (float)mn), 2.f), 128.f);
      const int cost = (mx - mn) + (int)fabsf(c);
      if (cost < best_cost) { best_cost = cost; best_r = r; }
    }
    if (lane == 0) rollings[img] = (int64_t)__fmul_rn(__fdiv_rn((float)best_r, 256.f), ref_w);
  }
}

// ---- (c) remap -----------------------------------------------------------------------------------------------
// A row is the contiguous run of Wo "units" that shares (b, c, y) (NCHW: unit = one element) or (b, y)
// (channels-last: unit = the C elements of a pixel).  Output unit x of image b reads input unit
//   sx = (ox_b + (flip ? Wo - 1 - x : x) - r_b) mod Wi   of input row  oy_b + y.
// Each thread writes 16 output bytes of one row: a 16-byte load when the source bytes are contiguous and
// aligned, byte moves otherwise (wrapped, flipped or misaligned chunks, and row edges).
struct RemapArgs {
  const uint8_t* in; uint8_t* out;
  int64_t B, C, Hi, Wi, Ho, Wo, unit, rows_per_img, row_bytes, chunks_per_row;
  const int64_t* rolls; const int64_t* offsets; int flip, channels_last;
};

__device__ __forceinline__ int64_t pmod(int64_t a, int64_t m) { const int64_t r = a % m; return r < 0 ? r + m : r; }

static __global__ void __launch_bounds__(256)
remap_kernel(RemapArgs a, int64_t total_chunks, int out_aligned) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total_chunks;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / a.chunks_per_row, k0 = (i - row * a.chunks_per_row) * 16;
    const int64_t b = row / a.rows_per_img, rr = row - b * a.rows_per_img;
    int64_t c, y;
    if (a.channels_last) { c = 0; y = rr; } else { c = rr / a.Ho; y = rr - c * a.Ho; }
    const int64_t r = a.rolls ? a.rolls[b] : 0;
    const int64_t ox = a.offsets ? a.offsets[2 * b] : 0, oy = a.offsets ? a.offsets[2 * b + 1] : 0;
    const int64_t sy = oy + y;
    uint8_t* dst = a.out + row * a.row_bytes + k0;
    const int64_t nb = min((int64_t)16, a.row_bytes - k0);
    if (sy < 0 || sy >= a.Hi) {                                   // offsets outside the map: zeros, no read
      for (int64_t j = 0; j < nb; ++j) dst[j] = 0;
      continue;
    }
    const int64_t in_row = a.channels_last ? (b * a.Hi + sy) : ((b * a.C + c) * a.Hi + sy);
    const uint8_t* src = a.in + in_row * a.Wi * a.unit;
    const int64_t x0 = k0 / a.unit, w0 = k0 - x0 * a.unit;
    const int64_t xf0 = a.flip ? a.Wo - 1 - x0 : x0;
    const int64_t s0 = pmod(ox + xf0 - r, a.Wi) * a.unit + w0;
    // contiguous source: no flip (or the chunk lies inside one unit) and no wrap inside the chunk
    const bool contiguous = (!a.flip || w0 + nb <= a.unit) && (s0 + nb <= a.Wi * a.unit);
    if (nb == 16 && out_aligned && contiguous && ((reinterpret_cast<uintptr_t>(src + s0) & 15u) == 0)) {
      *reinterpret_cast<uint4*>(dst) = __ldg(reinterpret_cast<const uint4*>(src + s0));
      continue;
    }
    // byte path: the source unit steps by +-1 with wrap-around (no division per byte)
    int64_t s = s0 / a.unit, w = w0;
    const int64_t ds = a.flip ? -1 : 1;
    auto next = [&]() {
      if (++w == a.unit) {
        w = 0; s += ds;
        if (s == a.Wi) s = 0; else if (s < 0) s = a.Wi - 1;
      }
    };
    if (nb == 16 && out_aligned) {                                // gather 16 bytes, one 16-byte store
      uint32_t word[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        word[j >> 2] |= (uint32_t)src[s * a.unit + w] << ((j & 3) * 8);
        next();
      }
      *reinterpret_cast<uint4*>(dst) = make_uint4(word[0], word[1], word[2], word[3]);
      continue;
    }
    for (int64_t j = 0; j < nb; ++j) {
      dst[j] = src[s * a.unit + w];
      next();
    }
  }
}

// ---- (d) coverage bookkeeping ----------------------------------------------------------------------------------
// Index (in the caller's workspace): image -> its points and point -> its images, both bucketed with
// bk::build_index.  The pick is a set operation, so the order inside a bucket does not matter.
struct CoverageIndex {
  bk::BucketIndex by_img, by_pt;
  int64_t *img_pts, *pt_imgs;
};

static size_t carve_coverage(uint8_t* base, int64_t V, int64_t n_img, int64_t N, CoverageIndex* w) {
  size_t o = 0;
  o += bk::carve_index(base, V, n_img, w ? &w->by_img : nullptr);
  o += bk::carve_index(base ? base + o : nullptr, V, N, w ? &w->by_pt : nullptr);
  if (w) w->img_pts = base ? (int64_t*)(base + o) : nullptr;
  o += round256((size_t)(V + 1) * 8);
  if (w) w->pt_imgs = base ? (int64_t*)(base + o) : nullptr;
  o += round256((size_t)(V + 1) * 8);
  return o;
}

struct KeyFrom { const int64_t* k; __device__ __forceinline__ void operator()(int64_t i, int64_t* out) const { out[0] = k[i]; } };

static __global__ void __launch_bounds__(256)
coverage_fill(const int64_t* __restrict__ gimg, const int64_t* __restrict__ vpoint, const int64_t* __restrict__ by_img,
              const int64_t* __restrict__ by_pt, int64_t V, int64_t* __restrict__ img_pts, int64_t* __restrict__ pt_imgs,
              const int64_t* __restrict__ img_off, int64_t n_img, int32_t* __restrict__ unseen,
              int32_t* __restrict__ seen, int64_t N) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < V; i += (int64_t)gridDim.x * blockDim.x) {
    img_pts[i] = vpoint[by_img[i]];
    pt_imgs[i] = gimg[by_pt[i]];
  }
  for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < n_img; g += (int64_t)gridDim.x * blockDim.x)
    unseen[g] = (int32_t)(img_off[g + 1] - img_off[g]);
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < N; p += (int64_t)gridDim.x * blockDim.x)
    seen[p] = 0;
}

// every point of image g seen for the first time takes one off the unseen count of every image that sees it
static __global__ void __launch_bounds__(256)
coverage_pick_kernel(int64_t g, const int64_t* __restrict__ img_off, const int64_t* __restrict__ img_pts,
                     const int64_t* __restrict__ pt_off, const int64_t* __restrict__ pt_imgs,
                     int32_t* __restrict__ seen, int32_t* __restrict__ unseen) {
  const int64_t k1 = img_off[g + 1];
  for (int64_t k = img_off[g] + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < k1;
       k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = img_pts[k];
    if (atomicExch(seen + p, 1) == 0)
      for (int64_t t = pt_off[p]; t < pt_off[p + 1]; ++t) atomicSub(unseen + pt_imgs[t], 1);
  }
}

}  // namespace dva

using namespace dva;

extern "C" int dva_mapping_image_stats(const int64_t* images, const int64_t* atomic_ptr, const void* pixels,
                                       int pix_code, int64_t V, int64_t n_img, int64_t ref_w, int64_t* count,
                                       int32_t* bbox, uint32_t* occ, void* stream) {
  if (V < 0 || n_img < 0) return fail(DVA_EINVAL, "mapping_image_stats: negative size");
  if (pix_code < 0 || pix_code > 2) return fail(DVA_EUNSUPPORTED, "mapping_image_stats: pixels must be int16/32/64");
  if (occ && ref_w <= 0) return fail(DVA_EINVAL, "mapping_image_stats: occupancy needs ref_w > 0");
  if (n_img == 0) return DVA_OK;
  if (!count || !bbox || (V > 0 && (!images || !atomic_ptr || !pixels)))
    return fail(DVA_EINVAL, "mapping_image_stats: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  stats_init<<<grid_cap(n_img, 256, 16), 256, 0, st>>>(count, bbox, occ, n_img);
  int rc = check_launch("mapping_image_stats_init");
  if (rc) return rc;
  if (V > 0) {
    const float rw = (float)ref_w;
    with_pix(pix_code, [&](auto p) {
      using PIX = decltype(p);
      stats_accumulate<PIX><<<grid_cap(V, 256, 16), 256, 0, st>>>(images, atomic_ptr, (const PIX*)pixels, V, n_img, rw,
                                                                  count, bbox, occ);
    });
    if ((rc = check_launch("mapping_image_stats"))) return rc;
  }
  stats_finalize<<<grid_cap(n_img, 256, 16), 256, 0, st>>>(count, bbox, n_img);
  return check_launch("mapping_image_stats_finalize");
}

extern "C" int dva_center_roll(const uint32_t* occ, int64_t n_img, int angular_res, int64_t ref_w, int64_t* rollings,
                               void* stream) {
  if (n_img < 0) return fail(DVA_EINVAL, "center_roll: negative size");
  if (angular_res < 1 || angular_res > 256) return fail(DVA_EINVAL, "center_roll: angular_res must be in [1, 256]");
  if (ref_w <= 0) return fail(DVA_EINVAL, "center_roll: ref_w must be positive");
  if (n_img == 0) return DVA_OK;
  if (!occ || !rollings) return fail(DVA_EINVAL, "center_roll: null pointer");
  center_roll_kernel<<<grid_cap(n_img * 32, 256, 16), 256, 0, (cudaStream_t)stream>>>(occ, n_img, 256 / angular_res,
                                                                          (float)ref_w, rollings);
  return check_launch("center_roll");
}

extern "C" int dva_image_remap(const void* in, void* out, int64_t B, int64_t C, int64_t Hi, int64_t Wi, int64_t Ho,
                               int64_t Wo, int elem_bytes, int channels_last, const int64_t* rolls,
                               const int64_t* offsets, int flip, void* stream) {
  if (B < 0 || C < 0 || Hi < 0 || Wi < 0 || Ho < 0 || Wo < 0) return fail(DVA_EINVAL, "image_remap: negative size");
  if (elem_bytes != 1 && elem_bytes != 2 && elem_bytes != 4)
    return fail(DVA_EUNSUPPORTED, "image_remap: element size must be 1, 2 or 4 bytes");
  if (Ho > Hi || Wo > Wi) return fail(DVA_EINVAL, "image_remap: output larger than the input");
  if (B == 0 || C == 0 || Ho == 0 || Wo == 0) return DVA_OK;
  if (!in || !out) return fail(DVA_EINVAL, "image_remap: null pointer");
  RemapArgs a;
  a.in = (const uint8_t*)in; a.out = (uint8_t*)out;
  a.B = B; a.C = C; a.Hi = Hi; a.Wi = Wi; a.Ho = Ho; a.Wo = Wo;
  a.unit = channels_last ? C * elem_bytes : elem_bytes;
  a.rows_per_img = channels_last ? Ho : C * Ho;
  a.row_bytes = Wo * a.unit;
  a.chunks_per_row = (a.row_bytes + 15) / 16;
  a.rolls = rolls; a.offsets = offsets; a.flip = flip ? 1 : 0; a.channels_last = channels_last ? 1 : 0;
  const int out_aligned = aligned16(out) && (a.row_bytes % 16 == 0);
  const int64_t total = B * a.rows_per_img * a.chunks_per_row;
  remap_kernel<<<grid_cap(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(a, total, out_aligned);
  return check_launch("image_remap");
}

extern "C" size_t dva_coverage_index_workspace_bytes(int64_t V, int64_t n_img, int64_t N) {
  if (V < 0 || n_img < 0 || N < 0) return 0;
  return carve_coverage(nullptr, V, n_img, N, nullptr);
}

extern "C" int dva_coverage_index(const int64_t* gimg, const int64_t* vpoint, int64_t V, int64_t n_img, int64_t N,
                                  int32_t* unseen, int32_t* seen, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  if (V < 0 || n_img < 0 || N < 0) return fail(DVA_EINVAL, "coverage_index: negative size");
  if (workspace_bytes < carve_coverage(nullptr, V, n_img, N, nullptr))
    return fail(DVA_EINVAL, "coverage_index: workspace too small");
  if (!workspace || (n_img > 0 && !unseen) || (N > 0 && !seen) || (V > 0 && (!gimg || !vpoint)))
    return fail(DVA_EINVAL, "coverage_index: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  CoverageIndex w;
  carve_coverage((uint8_t*)workspace, V, n_img, N, &w);
  int rc = bk::build_index<1>(KeyFrom{gimg}, V, n_img, w.by_img, st, /*order=*/false);
  if (rc) return rc;
  if ((rc = bk::build_index<1>(KeyFrom{vpoint}, V, N, w.by_pt, st, /*order=*/false))) return rc;
  coverage_fill<<<grid_cap(V > n_img ? (V > N ? V : N) : (n_img > N ? n_img : N), 256, 16), 256, 0, st>>>(
      gimg, vpoint, w.by_img.bucket, w.by_pt.bucket, V, w.img_pts, w.pt_imgs, w.by_img.off, n_img, unseen, seen, N);
  return check_launch("coverage_fill");
}

extern "C" int dva_coverage_pick(int64_t g, int64_t V, int64_t n_img, int64_t N, int32_t* unseen, int32_t* seen,
                                 const void* workspace, size_t workspace_bytes, void* stream) {
  if (V < 0 || n_img < 0 || N < 0) return fail(DVA_EINVAL, "coverage_pick: negative size");
  if (g < 0 || g >= n_img) return fail(DVA_EINVAL, "coverage_pick: image id out of range");
  if (workspace_bytes < carve_coverage(nullptr, V, n_img, N, nullptr))
    return fail(DVA_EINVAL, "coverage_pick: workspace too small");
  if (!workspace || !unseen || !seen) return fail(DVA_EINVAL, "coverage_pick: null pointer");
  CoverageIndex w;
  carve_coverage((uint8_t*)workspace, V, n_img, N, &w);
  coverage_pick_kernel<<<kNumSMs * 2, 256, 0, (cudaStream_t)stream>>>(g, w.by_img.off, w.img_pts, w.by_pt.off,
                                                                      w.pt_imgs, seen, unseen);
  return check_launch("coverage_pick");
}
