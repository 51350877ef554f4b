// Hand-written wgmma projection GEMMs of the pool MLPs (E_mod / E_mix / E_main; reference
// core/common_modules/base_modules.py:42 `nn.Linear(bias=False)` over ALL views, pooling.py:239-261).
//
//   rows kernel  (forward and dX):  D[M, N] = X[M, K] . W[N, K]^T      M = views (millions), N, K <= 512
//   dw kernel    (weight gradient): D[N, K] = dZ[M, N]^T . X[M, K]      contraction over the M rows
//
// Precision: 3xTF32.  Every fp32 operand is split x = hi + lo with hi = tf32(x) and lo = tf32(x - hi), both
// rounded to nearest (truncation would be a biased error that grows linearly with K); the tensor cores
// accumulate lo.hi + hi.lo + hi.hi in fp32 (the dropped lo.lo term is 2^-22 relative): fp32-grade results
// (~1e-6 of the result's max at K = 128, measured against fp64) at three TF32 MMAs per product.
//
// Both kernels are warp-specialised and persistent (one CTA per SM, 384 threads): warpgroup 0 is the TMA
// producer (one thread), warpgroups 1 and 2 are consumers that each own 64 rows of the 128 x 128 output tile
// and issue wgmma.m64n128k8 (tf32) with the A operand in REGISTERS and B from shared memory:
//   * A is read from the landed fp32 tile with plain shared loads and split into hi / lo in registers, so the
//     lo half never goes back to shared memory and the tensor core never sees an unsplit fp32 word;
//   * B is K-major in the SWIZZLE_128B canonical layout (rows of 32 fp32 = 128 bytes, 8-row atoms of 1024
//     bytes), the only layout wgmma reads for 32-bit types.  The rows kernel's B is the weight, pre-split by a
//     small prep kernel and TMA-loaded as is (resident for the whole kernel when K <= 128 and N <= 128, else
//     streamed per k-block next to X); the dw kernel's B is X^T, which the consumers transpose and split
//     from the landed tile into a double-buffered K-major hi / lo pair.
// Stages are handed over with mbarriers: full (TMA transaction count), empty (one arrival per consumer warp).
#include <cuda.h>

#include "dva_common.cuh"

namespace dva {
namespace tc {

constexpr int kTile = 128;                 // rows and columns of an output tile
constexpr int kBK = 32;                    // fp32 per k-block: one 128-byte swizzle row
constexpr int kTileBytes = kTile * kBK * 4;  // 16 KB
constexpr int kStages = 4;
constexpr int kThreads = 384;              // warpgroup 0: producer; warpgroups 1, 2: consumers
constexpr int kConsumerWarps = 8;

// ---- PTX wrappers ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  } while (!done);
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// barrier 1 over the 256 consumer threads (barrier 0 is __syncthreads)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous wgmma window
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] += A[64 x 8] (registers, tf32) . B[128 x 8]^T (shared-memory descriptor, tf32); one warpgroup
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1)
      : "memory");
}

// Shared-memory matrix descriptor of a K-major operand in the SWIZZLE_128B canonical layout: rows of 128
// bytes, 8-row atoms of 1024 bytes (stride byte offset), layout type 1 (128B swizzle) in bits 62-63.
// One k8 step of tf32 is 32 bytes along the row: +2 in the 16-byte address field.
__device__ __forceinline__ uint64_t smem_desc_k_sw128(uint32_t addr) {
  return (uint64_t)((addr >> 4) & 0x3fffu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// byte offset of fp32 element (r, c) in a [rows x 32] tile of that layout (what TMA writes with SWIZZLE_128B)
__device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return (uint32_t)(r * 128 + ((((c >> 2) ^ r) & 7) << 4) + (c & 3) * 4);
}

__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = tf32_rna(x);
  lo = tf32_rna(x - __uint_as_float(hi));
}

// A fragments of four k8 steps (32 fp32 columns of the k-block) for the 16 rows of this warp: a0 (g, t),
// a1 (g + 8, t), a2 (g, t + 4), a3 (g + 8, t + 4) of each step, g = lane / 4, t = lane % 4.  at(r, c) gives
// the fp32 element at tile row r, k-block column c.
template <typename At>
__device__ __forceinline__ void load_a_split(At at, int r, int t, uint32_t (&hi)[4][4], uint32_t (&lo)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    split_tf32(at(r, 8 * kk + t), hi[kk][0], lo[kk][0]);
    split_tf32(at(r + 8, 8 * kk + t), hi[kk][1], lo[kk][1]);
    split_tf32(at(r, 8 * kk + t + 4), hi[kk][2], lo[kk][2]);
    split_tf32(at(r + 8, 8 * kk + t + 4), hi[kk][3], lo[kk][3]);
  }
}

// 12 wgmma of one k-block (4 k8 steps x lo.hi, hi.lo, hi.hi); waits for them before returning
__device__ __forceinline__ void mma_kblock(float (&acc)[64], const uint32_t (&hi)[4][4], const uint32_t (&lo)[4][4],
                                           uint64_t b_hi, uint64_t b_lo) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t o = (uint64_t)(2 * kk);
    wgmma_tf32(acc, lo[kk], b_hi + o);
    wgmma_tf32(acc, hi[kk], b_lo + o);
    wgmma_tf32(acc, hi[kk], b_hi + o);
  }
  wgmma_commit();
  wgmma_wait_all();
  acc_fence(acc);
}

// ---- weight preparation: W [N, K] (or its transpose) -> hi / lo, rows zero-padded to a multiple of 128 ----
// transpose = 0: Wp[n, k] = W[n * ldw + k]      (forward: output column n, reduction k)
// transpose = 1: Wp[n, k] = W[k * ldw + n]      (dX: output column n = input channel, reduction k = out channel)
__global__ void __launch_bounds__(256)
split_weight_kernel(const float* __restrict__ W, float* __restrict__ hi, float* __restrict__ lo, int n_out,
                    int n_pad, int k_red, int64_t ldw, int transpose) {
  const int64_t total = (int64_t)n_pad * k_red;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(t / k_red), k = (int)(t - (int64_t)n * k_red);
    float w = 0.f;
    if (n < n_out) w = transpose ? W[(int64_t)k * ldw + n] : W[(int64_t)n * ldw + k];
    uint32_t h, l;
    split_tf32(w, h, l);
    hi[t] = __uint_as_float(h);
    lo[t] = __uint_as_float(l);
  }
}

// ---- rows kernel --------------------------------------------------------------------------------------------
struct RowsParams {
  float* out;            // [M, n_out] row-major, leading dimension ldo
  float* col_stats;      // nullptr or [gridDim.x, 3, 128] per-CTA (sum (v - shift), sum (v - shift)^2, shift) per column
  int64_t M;
  int n_out, n_tiles, k_blocks, ldo;
  int64_t m_tiles;
  int vec2;              // out rows and ldo allow 8-byte stores
};

// WRES = true : K <= 128 and one column tile: the split weight (hi, lo) is loaded once and stays resident in
//               shared memory (2 x 64 KB at most); the stages carry X only;
// WRES = false: wider layers: weight k-blocks are streamed through shared memory next to X.
template <bool WRES>
__global__ void __launch_bounds__(kThreads, 1)
tc_rows_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_whi,
               const __grid_constant__ CUtensorMap map_wlo, const RowsParams p) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment: swizzle atoms are addressed relative to 1024-byte boundaries
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int KB = p.k_blocks;
  constexpr uint32_t kStageBytes = (WRES ? 1u : 3u) * kTileBytes;   // X (, W_hi, W_lo)
  uint8_t* w_base = smem;                                          // WRES: W_hi k-blocks, then W_lo k-blocks
  uint8_t* st_base = smem + (WRES ? (size_t)2 * KB * kTileBytes : 0);
  uint64_t* bars = reinterpret_cast<uint64_t*>(st_base + kStages * kStageBytes);
  const uint32_t bar0 = smem_u32(bars);
  auto full = [&](int s) { return bar0 + 8u * s; };
  auto empty = [&](int s) { return bar0 + 8u * (kStages + s); };
  const uint32_t w_full = bar0 + 8u * (2 * kStages);
  // [consumer warp][2][128]: column sums of (v - shift), (v - shift)^2; each entry has exactly one writer
  double* stat = reinterpret_cast<double*>(bars + 2 * kStages + 1);
  float* shift = reinterpret_cast<float*>(stat + kConsumerWarps * 2 * kTile);   // [128]

  const int64_t tiles = p.m_tiles * p.n_tiles;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_x); tma_prefetch_desc(&map_whi); tma_prefetch_desc(&map_wlo);
    for (int s = 0; s < kStages; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), kConsumerWarps); }
    mbar_init(w_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = (int)threadIdx.x - 128; i >= 0 && i < kConsumerWarps * 2 * kTile; i += kThreads - 128) stat[i] = 0.0;
  __syncthreads();

  if (threadIdx.x < 128) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      if (WRES) {
        mbar_expect_tx(w_full, 2u * KB * kTileBytes);
        for (int kb = 0; kb < KB; ++kb) {
          tma_load_2d(smem_u32(w_base + (size_t)kb * kTileBytes), &map_whi, kb * kBK, 0, w_full);
          tma_load_2d(smem_u32(w_base + (size_t)(KB + kb) * kTileBytes), &map_wlo, kb * kBK, 0, w_full);
        }
      }
      int s = 0; uint32_t ph = 0;
      for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int64_t mt = t / p.n_tiles;
        const int nt = (int)(t - mt * p.n_tiles);
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(empty(s), ph ^ 1u);
          uint8_t* st = st_base + (size_t)s * kStageBytes;
          mbar_expect_tx(full(s), kStageBytes);
          tma_load_2d(smem_u32(st), &map_x, kb * kBK, (int)(mt * kTile), full(s));
          if (!WRES) {
            tma_load_2d(smem_u32(st + kTileBytes), &map_whi, kb * kBK, nt * kTile, full(s));
            tma_load_2d(smem_u32(st + 2 * kTileBytes), &map_wlo, kb * kBK, nt * kTile, full(s));
          }
          if (++s == kStages) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // ===================== consumers: 64 rows of the tile per warpgroup =====================
  const int ctid = threadIdx.x - 128, lane = threadIdx.x & 31;
  const int wg = ctid >> 7, w = (ctid >> 5) & 3, g = lane >> 2, q = lane & 3;
  const int ra = wg * 64 + w * 16 + g;                 // tile row of a0 / a2 and of d[4j], d[4j + 1]; + 8 for the others
  if (WRES) mbar_wait(w_full, 0);
  int s = 0; uint32_t ph = 0;
  bool first = true;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int64_t mt = t / p.n_tiles;
    const int nt = (int)(t - mt * p.n_tiles);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < KB; ++kb) {
      mbar_wait(full(s), ph);
      const uint8_t* xs = st_base + (size_t)s * kStageBytes;
      const uint8_t* whi = WRES ? w_base + (size_t)kb * kTileBytes : xs + kTileBytes;
      const uint8_t* wlo = WRES ? w_base + (size_t)(KB + kb) * kTileBytes : xs + 2 * kTileBytes;
      uint32_t ahi[4][4], alo[4][4];
      load_a_split([&](int r, int c) { return *reinterpret_cast<const float*>(xs + sw128_off(r, c)); }, ra, q, ahi, alo);
      mma_kblock(acc, ahi, alo, smem_desc_k_sw128(smem_u32(whi)), smem_desc_k_sw128(smem_u32(wlo)));
      __syncwarp();
      if (lane == 0) mbar_arrive(empty(s));           // X read into registers, the weight MMAs completed
      if (++s == kStages) { s = 0; ph ^= 1u; }
    }

    // ---- epilogue: registers -> global; thread owns rows r0, r0 + 8 and columns 8 j + 2 q + {0, 1} ----
    const int64_t r0 = mt * kTile + ra, r1 = r0 + 8;
    const int n0 = nt * kTile + 2 * q;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n = n0 + 8 * j;
      if (n >= p.n_out) continue;
      float* o0 = p.out + r0 * (int64_t)p.ldo + n;
      float* o1 = p.out + r1 * (int64_t)p.ldo + n;
      if (p.vec2 && n + 1 < p.n_out) {
        if (r0 < p.M) *reinterpret_cast<float2*>(o0) = make_float2(acc[4 * j], acc[4 * j + 1]);
        if (r1 < p.M) *reinterpret_cast<float2*>(o1) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      } else {
        if (r0 < p.M) o0[0] = acc[4 * j];
        if (r1 < p.M) o1[0] = acc[4 * j + 2];
        if (n + 1 < p.n_out) {
          if (r0 < p.M) o0[1] = acc[4 * j + 1];
          if (r1 < p.M) o1[1] = acc[4 * j + 3];
        }
      }
    }
    if (p.col_stats != nullptr) {
      // BatchNorm column statistics (single n tile): sums of (v - shift) and (v - shift)^2, shifted by row 0 of
      // this CTA's first tile (no catastrophic cancellation in the variance); per warp over its 16 rows, then
      // added in fp64 to the warp's own shared-memory slot by the one lane that owns the column (no atomics);
      // bn_stats_finalize_kernel recombines the CTAs in fp64
      if (first) {
        if (wg == 0 && w == 0 && g == 0) {
#pragma unroll
          for (int j = 0; j < 16; ++j) { shift[8 * j + 2 * q] = acc[4 * j]; shift[8 * j + 2 * q + 1] = acc[4 * j + 1]; }
        }
        consumers_sync();
        first = false;
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + 2 * q + e;
          const float sh = shift[c];
          const float d0 = r0 < p.M ? acc[4 * j + e] - sh : 0.f;
          const float d1 = r1 < p.M ? acc[4 * j + 2 + e] - sh : 0.f;
          float a = d0 + d1, b = fmaf(d0, d0, d1 * d1);
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
          }
          if (g == 0) {
            double* ws = stat + (ctid >> 5) * 2 * kTile;
            ws[c] += (double)a;
            ws[kTile + c] += (double)b;
          }
        }
      }
    }
  }
  if (p.col_stats != nullptr && p.n_tiles == 1) {
    consumers_sync();
    if (ctid < kTile) {
      double s1 = 0.0, s2 = 0.0;
      for (int wi = 0; wi < kConsumerWarps; ++wi) { s1 += stat[wi * 2 * kTile + ctid]; s2 += stat[wi * 2 * kTile + kTile + ctid]; }
      p.col_stats[((int64_t)blockIdx.x * 3 + 0) * kTile + ctid] = (float)s1;
      p.col_stats[((int64_t)blockIdx.x * 3 + 1) * kTile + ctid] = (float)s2;
      p.col_stats[((int64_t)blockIdx.x * 3 + 2) * kTile + ctid] = shift[ctid];
    }
  }
}

// ---- dw kernel: D[n_out, k_in] = sum over rows v of dZ[v, n_out] * X[v, k_in] --------------------------------
// Both operands have the contraction index v as their SLOW dimension.  A = dZ^T comes from registers, so any
// layout serves: it is read from the landed [32 rows x 128] dZ tile directly.  B = X^T must be K-major (v
// contiguous) in shared memory: the consumers transpose the landed X tile into that layout, splitting it into
// hi and lo on the way (two buffers, so the transposition of one row block overlaps the MMAs of the previous).
// One CTA = one (128 x 128 output tile, slice of the rows): it accumulates its slice in registers and writes a
// partial tile; dw_reduce_kernel adds the slices in a fixed order (deterministic, no atomics).
constexpr int kDwRows = 32;                      // contraction rows per stage
constexpr int kGroupBytes = kDwRows * 128;       // one [32 rows x 32 columns] TMA box
constexpr uint32_t kDwStageBytes = 2u * kTileBytes;   // dZ [32 x 128], X [32 x 128], four boxes each

struct DwParams {
  float* partial;        // [splits, n_pad, k_pad]
  int64_t V, blocks_total, blocks_per_split;
  int n_out, k_in, n_pad, k_pad, k_tiles, splits;
};

__global__ void __launch_bounds__(kThreads, 1)
tc_dw_kernel(const __grid_constant__ CUtensorMap map_dz, const __grid_constant__ CUtensorMap map_x, const DwParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* bt_base = smem + (size_t)kStages * kDwStageBytes;          // [2][hi, lo] X^T tiles, 16 KB each
  uint64_t* bars = reinterpret_cast<uint64_t*>(bt_base + 4 * kTileBytes);
  const uint32_t bar0 = smem_u32(bars);
  auto full = [&](int s) { return bar0 + 8u * s; };
  auto empty = [&](int s) { return bar0 + 8u * (kStages + s); };

  const int split = blockIdx.x % p.splits, tile = blockIdx.x / p.splits;
  const int nt = tile / p.k_tiles, kt = tile - nt * p.k_tiles;
  const int64_t b0 = (int64_t)split * p.blocks_per_split;
  int64_t b1 = b0 + p.blocks_per_split;
  if (b1 > p.blocks_total) b1 = p.blocks_total;
  const int64_t nblk = b1 > b0 ? b1 - b0 : 0;
  int a_groups = (p.n_out - nt * kTile + 31) / 32; if (a_groups > 4) a_groups = 4;
  int b_groups = (p.k_in - kt * kTile + 31) / 32; if (b_groups > 4) b_groups = 4;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_dz); tma_prefetch_desc(&map_x);
    for (int s = 0; s < kStages; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (threadIdx.x < 128) {
    if (threadIdx.x == 0) {
      int s = 0; uint32_t ph = 0;
      for (int64_t b = 0; b < nblk; ++b) {
        mbar_wait(empty(s), ph ^ 1u);
        uint8_t* st = smem + (size_t)s * kDwStageBytes;
        mbar_expect_tx(full(s), (uint32_t)(a_groups + b_groups) * kGroupBytes);
        const int row = (int)((b0 + b) * kDwRows);
        for (int gi = 0; gi < a_groups; ++gi)
          tma_load_2d(smem_u32(st + gi * kGroupBytes), &map_dz, nt * kTile + gi * 32, row, full(s));
        for (int gi = 0; gi < b_groups; ++gi)
          tma_load_2d(smem_u32(st + kTileBytes + gi * kGroupBytes), &map_x, kt * kTile + gi * 32, row, full(s));
        if (++s == kStages) { s = 0; ph ^= 1u; }
      }
    }
    return;
  }

  const int ctid = threadIdx.x - 128, lane = threadIdx.x & 31;
  const int wg = ctid >> 7, w = (ctid >> 5) & 3, g = lane >> 2, q = lane & 3;
  const int ra = wg * 64 + w * 16 + g;                 // output row (n_out index within the tile) of a0 / d[4j]
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  int s = 0; uint32_t ph = 0;
  for (int64_t b = 0; b < nblk; ++b) {
    mbar_wait(full(s), ph);
    const uint8_t* st = smem + (size_t)s * kDwStageBytes;
    uint8_t* bt_hi = bt_base + (size_t)(b & 1) * 2 * kTileBytes;
    uint8_t* bt_lo = bt_hi + kTileBytes;
    // X^T: element (column n, row v) of the landed box n / 32 -> row n, column v of the K-major hi / lo tiles;
    // a warp takes the 32 rows v of one column n (conflict-free 128-byte stores)
#pragma unroll 4
    for (int i = 0; i < kTile * kDwRows / 256; ++i) {
      const int e = i * 256 + ctid, v = e & 31, n = e >> 5;
      const float x = n < b_groups * 32
          ? *reinterpret_cast<const float*>(st + kTileBytes + (n >> 5) * kGroupBytes + sw128_off(v, n & 31)) : 0.f;
      uint32_t h, l;
      split_tf32(x, h, l);
      *reinterpret_cast<uint32_t*>(bt_hi + sw128_off(n, v)) = h;
      *reinterpret_cast<uint32_t*>(bt_lo + sw128_off(n, v)) = l;
    }
    // A = dZ^T: element (output row m, contraction row v) = dZ tile (v, m)
    uint32_t ahi[4][4], alo[4][4];
    load_a_split([&](int m, int v) {
      return m < a_groups * 32 ? *reinterpret_cast<const float*>(st + (m >> 5) * kGroupBytes + sw128_off(v, m & 31)) : 0.f;
    }, ra, q, ahi, alo);
    fence_proxy_async();                               // generic-proxy writes of X^T -> visible to wgmma
    consumers_sync();                                  // both halves of X^T written; MMAs of block b - 1 done
    __syncwarp();
    if (lane == 0) mbar_arrive(empty(s));             // the landed tiles are no longer read
    mma_kblock(acc, ahi, alo, smem_desc_k_sw128(smem_u32(bt_hi)), smem_desc_k_sw128(smem_u32(bt_lo)));
    if (++s == kStages) { s = 0; ph ^= 1u; }
  }
  // partial tile: rows nt * 128 + ra (+ 8), columns kt * 128 + 8 j + 2 q + {0, 1}
  float* d0 = p.partial + ((int64_t)split * p.n_pad + nt * kTile + ra) * p.k_pad + kt * kTile + 2 * q;
  float* d1 = d0 + 8 * (int64_t)p.k_pad;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    *reinterpret_cast<float2*>(d0 + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(d1 + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

__global__ void __launch_bounds__(256)
dw_reduce_kernel(const float* __restrict__ partial, float* __restrict__ out, int n_out, int k_in, int n_pad,
                 int k_pad, int splits, int64_t ldo) {
  const int64_t total = (int64_t)n_out * k_in;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(t / k_in), k = (int)(t - (int64_t)n * k_in);
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += partial[((int64_t)s * n_pad + n) * k_pad + k];   // fixed order
    out[(int64_t)n * ldo + k] = acc;
  }
}

// ---- BatchNorm statistics from the rows kernel's per-CTA partials (base_modules.py:44, nn.BatchNorm1d) ------
// One warp per column; lanes stride over the CTAs in a fixed order, fp64 combine:
//   sum_b = s_b + n_b sh_b,   sumsq_b = q_b + 2 sh_b s_b + n_b sh_b^2,   n_b = rows CTA b processed.
__global__ void __launch_bounds__(128)
bn_stats_finalize_kernel(const float* __restrict__ col_stats, int ctas, int64_t M, int64_t m_tiles, int C,
                         float eps, float momentum, float* __restrict__ mean, float* __restrict__ invstd,
                         float* __restrict__ running_mean, float* __restrict__ running_var) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  double S = 0.0, Q = 0.0;
  const int64_t rem = M - (m_tiles - 1) * kTile;       // rows of the globally last tile
  for (int b = lane; b < ctas; b += 32) {
    // tiles b, b + ctas, ...: all full except possibly the globally last one
    const int64_t nt = b < m_tiles ? (m_tiles - 1 - b) / ctas + 1 : 0;
    int64_t nb = nt * kTile;
    if (nt > 0 && b + (nt - 1) * ctas == m_tiles - 1) nb += rem - kTile;
    const double s = (double)col_stats[((int64_t)b * 3 + 0) * kTile + c];
    const double q = (double)col_stats[((int64_t)b * 3 + 1) * kTile + c];
    const double sh = (double)col_stats[((int64_t)b * 3 + 2) * kTile + c];
    S += s + (double)nb * sh;
    Q += q + 2.0 * sh * s + (double)nb * sh * sh;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { S += __shfl_xor_sync(0xffffffffu, S, o); Q += __shfl_xor_sync(0xffffffffu, Q, o); }
  if (lane != 0) return;
  const double n = (double)M, mu = S / n;
  double var = Q / n - mu * mu;
  if (var < 0.0) var = 0.0;
  mean[c] = (float)mu;
  invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean != nullptr) {
    const double unbiased = M > 1 ? var * n / (n - 1.0) : var;
    running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * mu);
    running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unbiased);
  }
}

// ---- host side ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    return (EncodeTiledFn)f;
  }();
  return fn;
}

// 2-D fp32 tensor [rows, cols] with leading dimension ld (elements); box = [box_rows x 32 columns], 128B swizzle
static int make_map(CUtensorMap* m, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return fail(DVA_EUNSUPPORTED, "tc_gemm: cuTensorMapEncodeTiled not available from the driver");
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return failf(DVA_EINVAL, "tc_gemm: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return DVA_OK;
}

static inline int n_pad_of(int64_t n_out) { return (int)((n_out + kTile - 1) / kTile) * kTile; }

}  // namespace tc
}  // namespace dva

using namespace dva;

// workspace of the rows kernel: split weight (hi | lo), rows padded to a multiple of 128
extern "C" size_t dva_tc_rows_workspace_bytes(int64_t n_out, int64_t k_red) {
  return (size_t)2 * tc::n_pad_of(n_out) * (size_t)k_red * 4 + 256;
}

extern "C" int dva_tc_rows_supported(int64_t M, int64_t n_out, int64_t k_red) {
  return M >= 1 && n_out >= 1 && k_red >= 4 && k_red % 4 == 0 && n_out <= 65536 && k_red <= 65536 && M < (1ll << 40);
}

// D[M, n_out] = X[M, k_red] . Wp^T with Wp[n, k] = transpose ? W[k, n] : W[n, k]   (W row-major, leading dimension ldw)
// col_stats: nullptr, or [kNumSMs, 3, 128] floats receiving the per-CTA shifted column statistics of D (n_out <= 128)
extern "C" int dva_tc_rows_gemm(const float* X, const float* W, float* D, int64_t M, int64_t n_out, int64_t k_red,
                                int64_t ldx, int64_t ldw, int64_t ldo, int transpose_w, float* col_stats,
                                int* stats_ctas, void* workspace, size_t workspace_bytes, void* stream) {
  if (M == 0) return DVA_OK;
  if (!dva_tc_rows_supported(M, n_out, k_red)) return fail(DVA_EUNSUPPORTED, "tc_rows_gemm: unsupported shape");
  if (!X || !W || !D || !workspace) return fail(DVA_EINVAL, "tc_rows_gemm: null pointer");
  if (!aligned16(X) || !aligned16(workspace) || ldx % 4 != 0) return fail(DVA_EALIGN, "tc_rows_gemm: X rows must be 16-byte aligned");
  if (workspace_bytes < dva_tc_rows_workspace_bytes(n_out, k_red)) return fail(DVA_EINVAL, "tc_rows_gemm: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int n_pad = tc::n_pad_of(n_out);
  float* whi = reinterpret_cast<float*>(workspace);
  float* wlo = whi + (size_t)n_pad * k_red;
  {
    const int64_t total = (int64_t)n_pad * k_red;
    tc::split_weight_kernel<<<grid_cap(total, 256, 4), 256, 0, st>>>(W, whi, wlo, (int)n_out, n_pad, (int)k_red, ldw, transpose_w);
    int rc = check_launch("split_weight");
    if (rc) return rc;
  }
  CUtensorMap mx, mh, ml;
  int rc = tc::make_map(&mx, X, M, k_red, ldx, tc::kTile);
  if (rc) return rc;
  rc = tc::make_map(&mh, whi, n_pad, k_red, k_red, tc::kTile);
  if (rc) return rc;
  rc = tc::make_map(&ml, wlo, n_pad, k_red, k_red, tc::kTile);
  if (rc) return rc;
  tc::RowsParams p;
  p.out = D; p.col_stats = col_stats; p.M = M; p.n_out = (int)n_out; p.n_tiles = n_pad / tc::kTile;
  p.k_blocks = (int)((k_red + tc::kBK - 1) / tc::kBK); p.ldo = (int)ldo; p.m_tiles = (M + tc::kTile - 1) / tc::kTile;
  p.vec2 = ldo % 2 == 0 && (reinterpret_cast<uintptr_t>(D) & 7u) == 0;
  const bool resident = p.n_tiles == 1 && p.k_blocks <= 4;
  if (col_stats && p.n_tiles != 1) return fail(DVA_EUNSUPPORTED, "tc_rows_gemm: column statistics need n_out <= 128");
  const int64_t tiles = p.m_tiles * p.n_tiles;
  const int grid = (int)(tiles < kNumSMs ? tiles : kNumSMs);
  if (stats_ctas) *stats_ctas = grid;
  const size_t smem = 1024 + (resident ? (size_t)(2 * p.k_blocks + tc::kStages) : (size_t)3 * tc::kStages) * tc::kTileBytes +
                      8 * (2 * tc::kStages + 1) + tc::kConsumerWarps * 2 * tc::kTile * 8 + tc::kTile * 4;
  cudaError_t e;
  if (resident) {
    e = cudaFuncSetAttribute(tc::tc_rows_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "tc_rows_gemm: cannot reserve shared memory");
    tc::tc_rows_kernel<true><<<grid, tc::kThreads, smem, st>>>(mx, mh, ml, p);
  } else {
    e = cudaFuncSetAttribute(tc::tc_rows_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "tc_rows_gemm: cannot reserve shared memory");
    tc::tc_rows_kernel<false><<<grid, tc::kThreads, smem, st>>>(mx, mh, ml, p);
  }
  return check_launch("tc_rows_gemm");
}

// ---- dW -------------------------------------------------------------------------------------------------------
static void dw_plan(int64_t V, int64_t n_out, int64_t k_in, int* n_tiles, int* k_tiles, int* splits, int64_t* bps,
                    int64_t* blocks) {
  *n_tiles = (int)((n_out + tc::kTile - 1) / tc::kTile);
  *k_tiles = (int)((k_in + tc::kTile - 1) / tc::kTile);
  *blocks = (V + tc::kDwRows - 1) / tc::kDwRows;
  int sp = kNumSMs / (*n_tiles * *k_tiles);
  if (sp < 1) sp = 1;
  if ((int64_t)sp > *blocks) sp = (int)(*blocks < 1 ? 1 : *blocks);
  *splits = sp;
  *bps = (*blocks + sp - 1) / sp;
}

extern "C" size_t dva_tc_dw_workspace_bytes(int64_t V, int64_t n_out, int64_t k_in) {
  int nt, kt, sp; int64_t bps, blocks;
  dw_plan(V, n_out, k_in, &nt, &kt, &sp, &bps, &blocks);
  return (size_t)sp * nt * tc::kTile * (size_t)kt * tc::kTile * 4 + 256;
}

// D[n_out, k_in] = dZ[V, n_out]^T . X[V, k_in]   (row-major, leading dimensions ldz / ldx / ldo)
extern "C" int dva_tc_dw_gemm(const float* dZ, const float* X, float* D, int64_t V, int64_t n_out, int64_t k_in,
                              int64_t ldz, int64_t ldx, int64_t ldo, void* workspace, size_t workspace_bytes,
                              void* stream) {
  if (n_out < 1 || k_in < 1 || V < 0 || n_out > 65536 || k_in > 65536) return fail(DVA_EUNSUPPORTED, "tc_dw_gemm: unsupported shape");
  if (!D || (V > 0 && (!dZ || !X)) || !workspace) return fail(DVA_EINVAL, "tc_dw_gemm: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (V == 0) {
    for (int64_t n = 0; n < n_out; ++n) {
      cudaError_t e = cudaMemsetAsync(D + n * ldo, 0, (size_t)k_in * 4, st);
      if (e != cudaSuccess) return fail((int)e, "tc_dw_gemm: memset failed");
    }
    return DVA_OK;
  }
  if (!aligned16(dZ) || !aligned16(X) || !aligned16(workspace) || ldz % 4 != 0 || ldx % 4 != 0)
    return fail(DVA_EALIGN, "tc_dw_gemm: operand rows must be 16-byte aligned");
  if (workspace_bytes < dva_tc_dw_workspace_bytes(V, n_out, k_in)) return fail(DVA_EINVAL, "tc_dw_gemm: workspace too small");
  tc::DwParams p;
  int nt, kt, sp; int64_t bps, blocks;
  dw_plan(V, n_out, k_in, &nt, &kt, &sp, &bps, &blocks);
  p.partial = reinterpret_cast<float*>(workspace);
  p.V = V; p.blocks_total = blocks; p.blocks_per_split = bps; p.n_out = (int)n_out; p.k_in = (int)k_in;
  p.n_pad = nt * tc::kTile; p.k_pad = kt * tc::kTile; p.k_tiles = kt; p.splits = sp;
  CUtensorMap mz, mx;
  int rc = tc::make_map(&mz, dZ, V, n_out, ldz, tc::kDwRows);
  if (rc) return rc;
  rc = tc::make_map(&mx, X, V, k_in, ldx, tc::kDwRows);
  if (rc) return rc;
  const size_t smem = 1024 + (size_t)tc::kStages * tc::kDwStageBytes + 4 * (size_t)tc::kTileBytes + 8 * 2 * tc::kStages;
  cudaError_t e = cudaFuncSetAttribute(tc::tc_dw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return fail((int)e, "tc_dw_gemm: cannot reserve shared memory");
  tc::tc_dw_kernel<<<nt * kt * sp, tc::kThreads, smem, st>>>(mz, mx, p);
  rc = check_launch("tc_dw_gemm");
  if (rc) return rc;
  const int64_t total = n_out * k_in;
  tc::dw_reduce_kernel<<<grid_cap(total, 256, 8), 256, 0, st>>>(
      p.partial, D, (int)n_out, (int)k_in, p.n_pad, p.k_pad, sp, ldo);
  return check_launch("tc_dw_reduce");
}

// Forward of one MLP layer's Linear with the BatchNorm batch statistics taken in the GEMM epilogue:
// D = X . W^T and mean / invstd (+ momentum update of the running buffers) of D's columns, without the
// separate statistics pass over D.  n_out <= 128 (one column tile) and not a skinny shape.
extern "C" size_t dva_linear_bnstats_workspace_bytes(int64_t n_out, int64_t k_red) {
  return dva_tc_rows_workspace_bytes(n_out, k_red) + (size_t)kNumSMs * 3 * tc::kTile * 4;
}

extern "C" int dva_tc_narrow();
extern "C" int dva_linear_bnstats_supported(int64_t M, int64_t n_out, int64_t k_red) {
  if (!(dva_tc_rows_supported(M, n_out, k_red) && n_out <= tc::kTile && n_out % 4 == 0)) return 0;
  if (dva_tc_narrow()) return n_out >= 32 && k_red >= 8;
  return n_out > 32 && k_red > 32;
}

extern "C" int dva_linear_bnstats_fwd(const float* X, const float* W, float* D, int64_t M, int64_t n_out,
                                      int64_t k_red, float eps, float momentum, float* mean, float* invstd,
                                      float* running_mean, float* running_var, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  if (!dva_linear_bnstats_supported(M, n_out, k_red)) return fail(DVA_EUNSUPPORTED, "linear_bnstats_fwd: unsupported shape");
  if (!mean || !invstd) return fail(DVA_EINVAL, "linear_bnstats_fwd: null pointer");
  if (workspace_bytes < dva_linear_bnstats_workspace_bytes(n_out, k_red)) return fail(DVA_EINVAL, "linear_bnstats_fwd: workspace too small");
  const size_t wbytes = dva_tc_rows_workspace_bytes(n_out, k_red);
  float* stats = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + wbytes);
  int ctas = 0;
  int rc = dva_tc_rows_gemm(X, W, D, M, n_out, k_red, k_red, k_red, n_out, 0, stats, &ctas, workspace, wbytes, stream);
  if (rc) return rc;
  tc::bn_stats_finalize_kernel<<<(int)((n_out + 3) / 4), 128, 0, (cudaStream_t)stream>>>(
      stats, ctas, M, (M + tc::kTile - 1) / tc::kTile, (int)n_out, eps, momentum, mean, invstd, running_mean,
      running_var);
  return check_launch("bn_stats_finalize");
}
