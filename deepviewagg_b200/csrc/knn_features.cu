// Neighbourhood-based mapping features (SURVEY §8(f) rank 2): the density and occlusion viewing
// conditions of NeighborhoodBasedMappingFeatures (core/data_transform/multimodal/image.py:431-612).
//
//   1. exact k-NN of every point among all points (:504-514: KeOps `argKmin` of the squared
//      distances; the FAISS branch is an approximate search and is not reproduced), or of a query
//      set among a separate search set (models/segmentation/multimodal/no3d.py:105-125, KeOps
//      `argmin` of the nearest seen point; a coarse block level bounds far queries) on a uniform
//      grid: points are counting-sorted by cell (host side: CUB sort through torch), one thread
//      per query walks cubic shells of cells outwards and stops as soon as its k-th best distance
//      is inside the visited cube.  Squared distances are (dx*dx + dy*dy) + dz*dz in fp32 without
//      FMA contraction; ties are ordered by point index, so the result is a deterministic
//      function of the input (the oracle restates exactly this order).
//   2. density (:521-546): (k+1) / (3.1416 d_k^2) / (1/voxel^2) per point, expanded to its views.
//   3. occlusion (:556-588): (1 + #neighbours seen by the same image) / (k+1) per view.  The
//      reference materialises a dense bool [n_points, n_images] table and k fancy-index gathers;
//      here a view scans the (short) image lists of its point's neighbours in the view CSR.
#include "dva_common.cuh"

namespace dva {

// k <= 64 keeps the 64-entry list per thread; 64 < k <= 128 uses a second instantiation with a
// 128-entry list (same search, twice the local-memory list)
constexpr int kKnnMax = 64;
constexpr int kKnnMaxWide = 128;
constexpr int kKnnMaxShells = 6;   // 13^3 cells; a query still open after that falls back (below)
constexpr int kKnnBlk = 8;         // fine cells per coarse block and axis (query / search case)

__global__ void __launch_bounds__(256)
knn_cell_ids_kernel(const float* __restrict__ xyz, int64_t* __restrict__ cell, int64_t n, float ox,
                    float oy, float oz, float inv_cs, int gx, int gy, int gz) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cx = min(max((int)floorf((xyz[3 * i + 0] - ox) * inv_cs), 0), gx - 1);
    const int cy = min(max((int)floorf((xyz[3 * i + 1] - oy) * inv_cs), 0), gy - 1);
    const int cz = min(max((int)floorf((xyz[3 * i + 2] - oz) * inv_cs), 0), gz - 1);
    cell[i] = ((int64_t)cz * gy + cy) * gx + cx;
  }
}

// (d2, id) lexicographic order
__device__ __forceinline__ bool knn_less(float d, int64_t i, float d2, int64_t i2) {
  return d < d2 || (d == d2 && i < i2);
}

// Search set: xyz_s / order_s in cell-sorted order (order_s[j] = original index of sorted slot j),
// cell_ptr [gx*gy*gz+1].  Queries: xyz_q / cell_q / order_q, also cell-sorted (neighbouring threads
// walk neighbouring cells); the self case passes the search arrays as the queries.
// Planar inputs (z = 0) give (dx*dx + dy*dy) + 0, the exact 2D squared distance.
//
// A query still open after kKnnMaxShells fine shells:
//   COARSE = false (self case): exhaustive scan of the search set;
//   COARSE = true  (query / search case): restarts on the coarse level, blocks of kKnnBlk^3 fine cells
//     with per-block counts blk_cnt [GZ*GY*GX].  Coarse shells of blocks are walked outwards from
//     the query's block; empty blocks are skipped, and so are blocks whose box lies farther than
//     the current k-th best.  It stops when the k-th best lies inside the lower bound of every
//     block outside the visited cube, or when no block is left: the search is exact either way.
// (the min-blocks hint of the coarse variant lets ptxas use 54 registers instead of spilling at 32)
template <int KMAX, bool COARSE>
__global__ void __launch_bounds__(128, COARSE ? 1 : 0)
knn_grid_kernel(const float* __restrict__ xyz_q, const int64_t* __restrict__ cell_q,
                const int64_t* __restrict__ order_q, int64_t nq, const float* __restrict__ xyz_s,
                const int64_t* __restrict__ order_s, const int64_t* __restrict__ cell_ptr, int64_t n,
                int k, float ox, float oy, float oz, float cs, int gx, int gy, int gz,
                const int* __restrict__ blk_cnt, int GX, int GY, int GZ,
                int64_t* __restrict__ nbr, float* __restrict__ d2out) {
  float bd[KMAX];
  int64_t bi[KMAX];
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < nq; q += (int64_t)gridDim.x * blockDim.x) {
    const float px = xyz_q[3 * q], py = xyz_q[3 * q + 1], pz = xyz_q[3 * q + 2];
    const int64_t c = cell_q[q];
    const int cx = (int)(c % gx), cy = (int)((c / gx) % gy), cz = (int)(c / ((int64_t)gx * gy));
    // distance from the query to the nearest face of its own cell (shell r adds r * cs); 0 for a
    // query outside the grid (clamped into a border cell), which keeps the bound conservative.  Faces
    // are measured from the same p - o the cell assignment used: o + cx * cs rounded at the ulp of |o|,
    // far more than the margin below once the cloud sits far from the origin (|o| ~ 1e5 m, 5 cm cells)
    const float rx = px - ox, ry = py - oy, rz = pz - oz;
    const float fx = rx - cx * cs, fy = ry - cy * cs, fz = rz - cz * cs;
    const float inner = fmaxf(fminf(fminf(fminf(fx, cs - fx), fminf(fy, cs - fy)), fminf(fz, cs - fz)), 0.f);
    int cnt = 0;
    auto offer = [&](float d2, int64_t id) {
      if (cnt == k && !knn_less(d2, id, bd[k - 1], bi[k - 1])) return;
      int t = (cnt < k) ? cnt : k - 1;                    // insertion into the sorted prefix
      while (t > 0 && knn_less(d2, id, bd[t - 1], bi[t - 1])) { bd[t] = bd[t - 1]; bi[t] = bi[t - 1]; --t; }
      bd[t] = d2; bi[t] = id;
      if (cnt < k) ++cnt;
    };
    // every search point of the x-row of cells [x0, x1] at (y, z)
    auto scan_row = [&](int z, int y, int x0, int x1) {
      const int64_t row = ((int64_t)z * gy + y) * gx;
      const int64_t j0 = cell_ptr[row + x0], j1 = cell_ptr[row + x1 + 1];
      for (int64_t j = j0; j < j1; ++j) {
        const float dx = __fsub_rn(px, xyz_s[3 * j]), dyy = __fsub_rn(py, xyz_s[3 * j + 1]),
                    dzz = __fsub_rn(pz, xyz_s[3 * j + 2]);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dyy, dyy)), __fmul_rn(dzz, dzz));
        offer(d2, order_s[j]);
      }
    };
    const int rmax = min(max(gx, max(gy, gz)), kKnnMaxShells);
    bool done = false;
    for (int r = 0; r <= rmax; ++r) {
      for (int dz = -r; dz <= r; ++dz) {
        const int z = cz + dz;
        if (z < 0 || z >= gz) continue;
        for (int dy = -r; dy <= r; ++dy) {
          const int y = cy + dy;
          if (y < 0 || y >= gy) continue;
          const bool face = (dz == -r || dz == r || dy == -r || dy == r);
          // a full x-row of cells on the shell's faces, else only its two end cells
          for (int part = 0; part < (face || r == 0 ? 1 : 2); ++part) {
            int x0, x1;
            if (face || r == 0) { x0 = cx - r; x1 = cx + r; }
            else { x0 = x1 = (part == 0 ? cx - r : cx + r); }
            if (x1 < 0 || x0 >= gx) continue;
            x0 = max(x0, 0); x1 = min(x1, gx - 1);
            scan_row(z, y, x0, x1);
          }
        }
      }
      if (cnt == k) {
        // everything outside the visited cube is farther than `reach` (margin for the rounding of
        // the cell assignment)
        const float reach = fmaxf(r * cs + inner - 1e-4f * cs, 0.f);
        if (bd[k - 1] <= reach * reach) { done = true; break; }
      }
    }
    if (!done && rmax < max(gx, max(gy, gz))) {
      if constexpr (COARSE) {
        // far query: restart on the coarse level (the blocks of shell R <= 1 contain the fine cube
        // already visited, so the restart costs at most that cube again)
        cnt = 0;
        const float bs = cs * kKnnBlk;
        const float margin = 1e-4f * cs;
        const int Cx = cx / kKnnBlk, Cy = cy / kKnnBlk, Cz = cz / kKnnBlk;
        const int Rmax = max(GX, max(GY, GZ));
        // lower bound of the distance from the query to [lo, lo + bs) on one axis, shrunk by the
        // cell-assignment margin and by a relative 1e-5 for the rounding of far distances
        // (p and lo relative to the grid origin, as the fine level's faces)
        auto gap = [&](float p, float lo) {
          const float g = fmaxf(fmaxf(lo - p, p - (lo + bs)), 0.f);
          return fmaxf(g - 1e-5f * g - margin, 0.f);
        };
        for (int R = 0; R <= Rmax; ++R) {
          for (int bz = Cz - R; bz <= Cz + R; ++bz) {
            if (bz < 0 || bz >= GZ) continue;
            for (int by = Cy - R; by <= Cy + R; ++by) {
              if (by < 0 || by >= GY) continue;
              const bool face = (bz == Cz - R || bz == Cz + R || by == Cy - R || by == Cy + R);
              const int step = (face || R == 0) ? 1 : 2 * R;     // interior rows: the two end blocks
              for (int bx = Cx - R; bx <= Cx + R; bx += step) {
                if (bx < 0 || bx >= GX) continue;
                if (blk_cnt[((int64_t)bz * GY + by) * GX + bx] == 0) continue;
                if (cnt == k) {
                  const float ax = gap(rx, bx * bs), ay = gap(ry, by * bs), az = gap(rz, bz * bs);
                  if (__fadd_rn(__fadd_rn(__fmul_rn(ax, ax), __fmul_rn(ay, ay)), __fmul_rn(az, az)) > bd[k - 1])
                    continue;
                }
                const int x0 = bx * kKnnBlk, x1 = min(x0 + kKnnBlk, gx) - 1;
                for (int z = bz * kKnnBlk; z < min(bz * kKnnBlk + kKnnBlk, gz); ++z)
                  for (int y = by * kKnnBlk; y < min(by * kKnnBlk + kKnnBlk, gy); ++y) scan_row(z, y, x0, x1);
              }
            }
          }
          if (cnt == k) {
            // nearest face of the visited block cube that has blocks beyond it
            float reach = INFINITY;
            if (Cx - R > 0) reach = fminf(reach, rx - (Cx - R) * bs);
            if (Cx + R + 1 < GX) reach = fminf(reach, (Cx + R + 1) * bs - rx);
            if (Cy - R > 0) reach = fminf(reach, ry - (Cy - R) * bs);
            if (Cy + R + 1 < GY) reach = fminf(reach, (Cy + R + 1) * bs - ry);
            if (Cz - R > 0) reach = fminf(reach, rz - (Cz - R) * bs);
            if (Cz + R + 1 < GZ) reach = fminf(reach, (Cz + R + 1) * bs - rz);
            if (reach == INFINITY) break;                        // every block visited
            reach = fmaxf(reach - 1e-5f * reach - margin, 0.f);
            if (bd[k - 1] <= reach * reach) break;
          }
        }
      } else {
        // isolated point (outlier, or a cell size far too small here): exhaustive scan
        cnt = 0;
        for (int64_t j = 0; j < n; ++j) {
          const float dx = __fsub_rn(px, xyz_s[3 * j]), dyy = __fsub_rn(py, xyz_s[3 * j + 1]),
                      dzz = __fsub_rn(pz, xyz_s[3 * j + 2]);
          offer(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dyy, dyy)), __fmul_rn(dzz, dzz)), order_s[j]);
        }
      }
    }
    const int64_t me = order_q[q];
    for (int t = 0; t < k; ++t) {
      nbr[me * k + t] = (t < cnt) ? bi[t] : -1;
      if (d2out != nullptr) d2out[me * k + t] = (t < cnt) ? bd[t] : INFINITY;
    }
  }
}

// one thread per view: density of its point + occlusion of the view, for every k in klist
__global__ void __launch_bounds__(256)
neighborhood_features_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ nbr, int kmax,
                             const int64_t* __restrict__ vptr, const int64_t* __restrict__ images,
                             const int64_t* __restrict__ view_point, const int* __restrict__ klist,
                             int nk, float voxel_density, int do_density, int do_occlusion,
                             float* __restrict__ out, int64_t V) {
  const int width = (do_density ? nk : 0) + (do_occlusion ? nk : 0);
  for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < V; v += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = view_point[v];
    float* __restrict__ o = out + v * width;
    int col = 0;
    if (do_density) {
      const float px = xyz[3 * p], py = xyz[3 * p + 1], pz = xyz[3 * p + 2];
      for (int a = 0; a < nk; ++a) {
        const int k = klist[a];
        const int64_t q = nbr[p * kmax + (k - 1)];
        // d2_max = ((xyz - xyz[neighbors[:, k-1]])**2).sum(1)                    :527
        const float dx = __fsub_rn(px, xyz[3 * q]), dy = __fsub_rn(py, xyz[3 * q + 1]), dz = __fsub_rn(pz, xyz[3 * q + 2]);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        // density = ((k+1) / (3.1416 d2)) / (1/voxel^2); NaN -> 1                :532-537
        float den = __fdiv_rn(__fdiv_rn((float)(k + 1), __fmul_rn(3.1416f, d2)), voxel_density);
        if (den != den) den = 1.f;
        o[col++] = den;
      }
    }
    if (do_occlusion) {
      const int64_t img = images[v];
      float seen = 1.f;                                   // the point itself                :575
      int a = 0;
      for (int i = 0; i < kmax && a < nk; ++i) {
        const int64_t q = nbr[p * kmax + i];
        bool hit = false;
        for (int64_t w = vptr[q]; w < vptr[q + 1]; ++w) hit |= (images[w] == img);
        seen += hit ? 1.f : 0.f;
        while (a < nk && klist[a] == i + 1) { o[col + a] = __fdiv_rn(seen, (float)(klist[a] + 1)); ++a; }   // :584
      }
    }
  }
}

}  // namespace dva

using namespace dva;

extern "C" int dva_knn_cell_ids(const float* xyz, int64_t* cell, int64_t n, float ox, float oy, float oz,
                                float cell_size, int gx, int gy, int gz, void* stream) {
  if (n < 0 || gx < 1 || gy < 1 || gz < 1 || !(cell_size > 0.f)) return fail(DVA_EINVAL, "knn_cell_ids: bad sizes");
  if (n == 0) return DVA_OK;
  if (!xyz || !cell) return fail(DVA_EINVAL, "knn_cell_ids: null pointer");
  knn_cell_ids_kernel<<<grid_cap(n, 256, 16), 256, 0, (cudaStream_t)stream>>>(xyz, cell, n, ox, oy, oz, 1.f / cell_size, gx, gy, gz);
  return check_launch("knn_cell_ids");
}

extern "C" int dva_knn_grid(const float* xyz_sorted, const int64_t* cell_sorted, const int64_t* order,
                            const int64_t* cell_ptr, int64_t n, int k, float ox, float oy, float oz,
                            float cell_size, int gx, int gy, int gz, int64_t* neighbors, float* dist2,
                            void* stream) {
  if (n < 0 || gx < 1 || gy < 1 || gz < 1 || !(cell_size > 0.f)) return fail(DVA_EINVAL, "knn_grid: bad sizes");
  if (k < 1 || k > kKnnMaxWide) return fail(DVA_EUNSUPPORTED, "knn_grid: k must be in [1, 128]");
  if (n == 0) return DVA_OK;
  if (!xyz_sorted || !cell_sorted || !order || !cell_ptr || !neighbors) return fail(DVA_EINVAL, "knn_grid: null pointer");
  // the self case: the search set is its own query set
  if (k <= kKnnMax)
    knn_grid_kernel<kKnnMax, false><<<grid_cap(n, 128, 16), 128, 0, (cudaStream_t)stream>>>(
        xyz_sorted, cell_sorted, order, n, xyz_sorted, order, cell_ptr, n, k, ox, oy, oz, cell_size, gx, gy, gz,
        nullptr, 0, 0, 0, neighbors, dist2);
  else
    knn_grid_kernel<kKnnMaxWide, false><<<grid_cap(n, 128, 16), 128, 0, (cudaStream_t)stream>>>(
        xyz_sorted, cell_sorted, order, n, xyz_sorted, order, cell_ptr, n, k, ox, oy, oz, cell_size, gx, gy, gz,
        nullptr, 0, 0, 0, neighbors, dist2);
  return check_launch("knn_grid");
}

extern "C" int dva_knn_query(const float* query_sorted, const int64_t* query_cell_sorted, const int64_t* query_order,
                             int64_t nq, const float* search_sorted, const int64_t* search_order,
                             const int64_t* cell_ptr, const int32_t* block_counts, int64_t ns, int k, float ox,
                             float oy, float oz, float cell_size, int gx, int gy, int gz, int64_t* neighbors,
                             float* dist2, void* stream) {
  if (nq < 0 || ns < 0 || gx < 1 || gy < 1 || gz < 1 || !(cell_size > 0.f))
    return fail(DVA_EINVAL, "knn_query: bad sizes");
  if (k < 1 || k > kKnnMaxWide) return fail(DVA_EUNSUPPORTED, "knn_query: k must be in [1, 128]");
  if (nq == 0) return DVA_OK;
  if (ns < k) return fail(DVA_EINVAL, "knn_query: the search set has fewer than k points");
  if (!query_sorted || !query_cell_sorted || !query_order || !search_sorted || !search_order || !cell_ptr ||
      !block_counts || !neighbors)
    return fail(DVA_EINVAL, "knn_query: null pointer");
  const int GX = (gx + kKnnBlk - 1) / kKnnBlk, GY = (gy + kKnnBlk - 1) / kKnnBlk, GZ = (gz + kKnnBlk - 1) / kKnnBlk;
  if (k <= kKnnMax)
    knn_grid_kernel<kKnnMax, true><<<grid_cap(nq, 128, 16), 128, 0, (cudaStream_t)stream>>>(
        query_sorted, query_cell_sorted, query_order, nq, search_sorted, search_order, cell_ptr, ns, k, ox, oy, oz,
        cell_size, gx, gy, gz, block_counts, GX, GY, GZ, neighbors, dist2);
  else
    knn_grid_kernel<kKnnMaxWide, true><<<grid_cap(nq, 128, 16), 128, 0, (cudaStream_t)stream>>>(
        query_sorted, query_cell_sorted, query_order, nq, search_sorted, search_order, cell_ptr, ns, k, ox, oy, oz,
        cell_size, gx, gy, gz, block_counts, GX, GY, GZ, neighbors, dist2);
  return check_launch("knn_query");
}

extern "C" int dva_neighborhood_features(const float* xyz, const int64_t* neighbors, int kmax,
                                         const int64_t* view_ptr, const int64_t* images,
                                         const int64_t* view_point, const int32_t* klist, int nk,
                                         double voxel, int density, int occlusion, float* out,
                                         int64_t N, int64_t V, void* stream) {
  if (N < 0 || V < 0 || kmax < 1 || nk < 1) return fail(DVA_EINVAL, "neighborhood_features: bad sizes");
  if (!density && !occlusion) return fail(DVA_EINVAL, "neighborhood_features: nothing to compute");
  if (V == 0) return DVA_OK;
  if (!xyz || !neighbors || !view_ptr || !images || !view_point || !klist || !out)
    return fail(DVA_EINVAL, "neighborhood_features: null pointer");
  // voxel_density = 1 / voxel**2 evaluated in double, then used as an fp32 scalar            :531
  const float voxel_density = (float)(1.0 / (voxel * voxel));
  neighborhood_features_kernel<<<grid_cap(V, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      xyz, neighbors, kmax, view_ptr, images, view_point, klist, nk, voxel_density, density, occlusion, out, V);
  return check_launch("neighborhood_features");
}
