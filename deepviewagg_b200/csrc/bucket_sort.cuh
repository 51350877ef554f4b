// Stable counting sort of items into dense integer buckets, shared by the mapping build
// (csrc/mapping_build.cu: items bucketed by point) and the deterministic backward passes
// (csrc/gather_pool.cu: map-gradient contributions bucketed by feature-map pixel;
// csrc/segment_csr.cu: source rows bucketed by destination row).
//
//   histogram (count_keys) -> exclusive scan (exclusive_scan) -> scatter (scatter_keys) -> order
//
// The scatter claims slots with atomics, so the order inside a bucket is arbitrary; one warp per
// bucket then rank-sorts it (warp_rank_sort).  With the entry id as the last key the result equals
// a STABLE sort and is a pure function of the input, whatever the launch configuration.
#pragma once
#include "dva_common.cuh"

namespace dva {
namespace bk {

constexpr int kScanItems = 2048;          // elements per scan block (256 threads x 8)

// ---- exclusive scan int32 -> int64 (three phases; sizes up to 2^31 blocks of 2048) -------------------
static __global__ void __launch_bounds__(256)
scan_block_sums(const int32_t* __restrict__ in, int64_t n, int64_t* __restrict__ block_sums) {
  __shared__ int64_t red[8];
  const int64_t base = (int64_t)blockIdx.x * kScanItems;
  int64_t s = 0;
  for (int k = 0; k < 8; ++k) {
    const int64_t i = base + k * 256 + threadIdx.x;
    if (i < n) s += in[i];
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t t = 0;
    for (int w = 0; w < 8; ++w) t += red[w];
    block_sums[blockIdx.x] = t;
  }
}

// single CTA: exclusive scan of the block sums in place; total -> sums[n_blocks]
static __global__ void __launch_bounds__(1024)
scan_of_sums(int64_t* __restrict__ sums, int64_t n_blocks) {
  __shared__ int64_t warp_tot[32];
  __shared__ int64_t carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int64_t base = 0; base < n_blocks; base += 1024) {
    const int64_t i = base + threadIdx.x;
    const int64_t v = i < n_blocks ? sums[i] : 0;
    int64_t inc = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t t = __shfl_up_sync(0xffffffffu, inc, o);
      if ((threadIdx.x & 31) >= o) inc += t;
    }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = inc;
    __syncthreads();
    if (threadIdx.x < 32) {
      int64_t w = warp_tot[threadIdx.x], wi = w;
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t t = __shfl_up_sync(0xffffffffu, wi, o);
        if (threadIdx.x >= o) wi += t;
      }
      warp_tot[threadIdx.x] = wi - w;                  // exclusive prefix of the warp totals
    }
    __syncthreads();
    const int64_t carry = carry_s;
    if (i < n_blocks) sums[i] = carry + warp_tot[threadIdx.x >> 5] + inc - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + warp_tot[31] + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) sums[n_blocks] = carry_s;
}

static __global__ void __launch_bounds__(256)
scan_apply(const int32_t* __restrict__ in, int64_t n, const int64_t* __restrict__ block_offsets,
           int64_t* __restrict__ out /* [n + 1] */) {
  __shared__ int64_t warp_tot[8];
  const int64_t base = (int64_t)blockIdx.x * kScanItems + (int64_t)threadIdx.x * 8;
  int32_t v[8];
  int64_t s = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) { v[k] = (base + k < n) ? in[base + k] : 0; s += v[k]; }
  int64_t inc = s;
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if ((threadIdx.x & 31) >= o) inc += t;
  }
  if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = inc;
  __syncthreads();
  int64_t pre = block_offsets[blockIdx.x] + inc - s;
  for (int w = 0; w < (threadIdx.x >> 5); ++w) pre += warp_tot[w];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (base + k < n) out[base + k] = pre;
    pre += v[k];
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) out[n] = block_offsets[gridDim.x];
}

static inline int64_t scan_block_words(int64_t n) { return (n + kScanItems - 1) / kScanItems + 2; }

static int exclusive_scan(const int32_t* in, int64_t n, int64_t* out, int64_t* block_sums, cudaStream_t st) {
  // out[0..n] = exclusive prefix sums of in[0..n), out[n] = total.  block_sums: scan_block_words(n) words
  if (n == 0) {
    cudaError_t e = cudaMemsetAsync(out, 0, 8, st);
    return e == cudaSuccess ? DVA_OK : fail((int)e, "scan: memset failed");
  }
  const int64_t nb = (n + kScanItems - 1) / kScanItems;
  scan_block_sums<<<(unsigned)nb, 256, 0, st>>>(in, n, block_sums);
  int rc = check_launch("scan_block_sums");
  if (rc) return rc;
  scan_of_sums<<<1, 1024, 0, st>>>(block_sums, nb);
  if ((rc = check_launch("scan_of_sums"))) return rc;
  scan_apply<<<(unsigned)nb, 256, 0, st>>>(in, n, block_sums, out);
  return check_launch("scan_apply");
}

// ---- bucketing -----------------------------------------------------------------------------------------
// key_of(i, k) writes the NK bucket keys of item i into k[0..NK); entry i * NK + j goes to bucket k[j].
// A key outside [0, nb) drops that entry (the functor may record it).
template <int NK, typename KeyOf>
__global__ void __launch_bounds__(256)
count_keys(KeyOf key_of, int64_t n, int64_t nb, int32_t* __restrict__ cnt) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t k[NK];
    key_of(i, k);
#pragma unroll
    for (int j = 0; j < NK; ++j)
      if (k[j] >= 0 && k[j] < nb) atomicAdd(cnt + k[j], 1);
  }
}

template <int NK, typename KeyOf>
__global__ void __launch_bounds__(256)
scatter_keys(KeyOf key_of, int64_t n, int64_t nb, const int64_t* __restrict__ off, int32_t* __restrict__ cursor,
             int64_t* __restrict__ bucket) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t k[NK];
    key_of(i, k);
#pragma unroll
    for (int j = 0; j < NK; ++j)       // arbitrary order inside the bucket; ordered next
      if (k[j] >= 0 && k[j] < nb) bucket[off[k[j]] + atomicAdd(cursor + k[j], 1)] = i * NK + j;
  }
}

// ---- ordering inside a bucket ----------------------------------------------------------------------------
// sort key of an entry: a, then the entry id (stability)
struct Key { int64_t a; int64_t src; };
__device__ __forceinline__ bool key_less(const Key& u, const Key& v) { return u.a < v.a || (u.a == v.a && u.src < v.src); }

// One warp: sorted[b0 + rank] = bucket[b0 + i] ordered by make_key(entry).  Buckets of up to 32 entries
// rank in registers (one shuffle round per entry); larger ones re-read the bucket per lane (L1 / L2).
// All 32 lanes must call it; the caller __syncwarp()s before reading `sorted`.
template <typename MakeKey>
__device__ __forceinline__ void warp_rank_sort(const int64_t* __restrict__ bucket, int64_t* __restrict__ sorted,
                                               int64_t b0, int64_t L, int lane, MakeKey make_key) {
  if (L <= 32) {
    Key mine; mine.a = 0; mine.src = 0;
    if (lane < L) mine = make_key(bucket[b0 + lane]);
    int rank = 0;
    for (int j = 0; j < (int)L; ++j) {
      Key o; o.a = __shfl_sync(0xffffffffu, mine.a, j); o.src = __shfl_sync(0xffffffffu, mine.src, j);
      rank += key_less(o, mine) ? 1 : 0;
    }
    if (lane < L) sorted[b0 + rank] = mine.src;
  } else {
    for (int64_t i = lane; i < L; i += 32) {
      const Key mine = make_key(bucket[b0 + i]);
      int64_t rank = 0;
      for (int64_t j = 0; j < L; ++j) rank += key_less(make_key(bucket[b0 + j]), mine) ? 1 : 0;
      sorted[b0 + rank] = mine.src;
    }
  }
}

// One warp per bucket: entries in ascending id.
struct IdKey { __device__ __forceinline__ Key operator()(int64_t e) const { Key k; k.a = 0; k.src = e; return k; } };
static __global__ void __launch_bounds__(256)
order_by_id(const int64_t* __restrict__ off, const int64_t* __restrict__ bucket, int64_t* __restrict__ sorted,
            int64_t nb) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < nb; q += warps) {
    const int64_t b0 = off[q], L = off[q + 1] - b0;
    if (L == 0) continue;
    if (L == 1) { if (lane == 0) sorted[b0] = bucket[b0]; continue; }
    warp_rank_sort(bucket, sorted, b0, L, lane, IdKey{});
  }
}

// ---- the whole index: off [nb + 1] (bucket q holds sorted[off[q] .. off[q+1])) ----------------------------
struct BucketIndex {
  int32_t *cnt, *cursor;            // [nb + 1] each, contiguous (one memset)
  int64_t *off, *block_sums, *bucket, *sorted;
};

// carves the index out of base (nullptr: size query); returns the bytes used
static size_t carve_index(uint8_t* base, int64_t n_entries, int64_t nb, BucketIndex* w) {
  size_t o = 0;
  auto take = [&](size_t bytes) { uint8_t* p = base ? base + o : nullptr; o += round256(bytes); return p; };
  uint8_t* p;
  p = take((size_t)(nb + 1) * 8); if (w) { w->cnt = (int32_t*)p; w->cursor = w->cnt ? w->cnt + (nb + 1) : nullptr; }
  p = take((size_t)(nb + 1) * 8); if (w) w->off = (int64_t*)p;
  p = take((size_t)scan_block_words(nb) * 8); if (w) w->block_sums = (int64_t*)p;
  p = take((size_t)(n_entries + 1) * 8); if (w) w->bucket = (int64_t*)p;
  p = take((size_t)(n_entries + 1) * 8); if (w) w->sorted = (int64_t*)p;
  return o;
}

// n_items items of NK entries each -> stable bucket index in w.sorted (w carved by carve_index).  With
// order == false the ordering pass is skipped and the caller reads w.bucket, whose order inside a bucket is
// arbitrary: for uses that treat a bucket as a set.
template <int NK, typename KeyOf>
static int build_index(KeyOf key_of, int64_t n_items, int64_t nb, const BucketIndex& w, cudaStream_t st,
                       bool order = true) {
  cudaError_t e = cudaMemsetAsync(w.cnt, 0, (size_t)(nb + 1) * 8, st);       // cnt + cursor
  if (e != cudaSuccess) return fail((int)e, "bucket index: memset failed");
  int rc;
  if (n_items > 0) {
    count_keys<NK><<<grid_cap(n_items, 256, 16), 256, 0, st>>>(key_of, n_items, nb, w.cnt);
    if ((rc = check_launch("bucket_count_keys"))) return rc;
  }
  if ((rc = exclusive_scan(w.cnt, nb, w.off, w.block_sums, st))) return rc;
  if (n_items > 0) {
    scatter_keys<NK><<<grid_cap(n_items, 256, 16), 256, 0, st>>>(key_of, n_items, nb, w.off, w.cursor, w.bucket);
    if ((rc = check_launch("bucket_scatter_keys"))) return rc;
    if (!order) return DVA_OK;
    order_by_id<<<grid_cap(nb * 32, 256, 16), 256, 0, st>>>(w.off, w.bucket, w.sorted, nb);
    if ((rc = check_launch("bucket_order_by_id"))) return rc;
  }
  return DVA_OK;
}

}  // namespace bk
}  // namespace dva
