// Segmentation evaluation (libdva_eval.so, C ABI include/dva_eval.h): the confusion update of the reference's
// trackers, their vote table and the full-resolution nearest-neighbour prediction.
//
//   confusion_scores_kernel<T>  argmax of each score row in registers (numpy's rule: the first index of the
//        maximum, the first NaN wins), counted into a per-CTA K x K int32 histogram in shared memory (equal
//        cells of a warp are added once, through __match_any_sync), then added to the int64 matrix with
//        integer atomics: the matrix does not depend on the order of the additions.  Neither the [n] argmax
//        nor a masked copy of the rows exists.
//   confusion_pred_kernel  the same from int64 predictions.
//   vote_claim_kernel + vote_add_kernel<T>  votes[ids] += outputs; counts[ids] += 1.  torch's index_put_
//        leaves the result of a duplicated id undefined; here the last occurrence wins: the claim pass takes
//        atomicMax(stamp[id], j), the add pass lets the owner j add its row (one __fadd_rn per element, the
//        bits of torch's votes + outputs), bump the count and put the stamp back to -1.  No pass touches the
//        whole table.
//   nn_vote_kernel  knn_interpolate(k = 1) + argmax + confusion, fused: for each query the row of its nearest
//        voted point, in torch_geometric's fp32 order (diff = pos_x - pos_y, d2 = (dx dx + dy dy) + dz dz,
//        w = 1 / max(d2, 1e-16), y = (x w) / w, every step rounded on its own), so a near-tie flips exactly
//        as it does there.  The [N_full, K] interpolated tensor never exists.
//
// Range errors (labels, predictions, ids) are not counted: they OR a DVA_EVAL_BAD_* bit into the caller's
// device status word, which nothing here reads back.
#include "dva_common.cuh"
#include "../../include/dva_eval.h"

// namespace dva_eval: the kernels of libdva_eval.so (case table: tests/test_eval_matrix_table.py)
namespace dva_eval {
using namespace dva;

constexpr int kEvThreads = 256;
constexpr int kEvMaxK = DVA_EVAL_MAX_CLASSES;

// numpy's argmax of get(0 .. K-1): the first index of the maximum; the first NaN wins
template <typename G> __device__ __forceinline__ int argmax_first(int K, G get) {
  float best = get(0);
  if (isnan(best)) return 0;
  int arg = 0;
  for (int c = 1; c < K; ++c) {
    const float v = get(c);
    if (isnan(v)) return c;
    if (v > best) { best = v; arg = c; }
  }
  return arg;
}

__device__ __forceinline__ void hist_zero(int* sh, int cells) {
  for (int c = threadIdx.x; c < cells; c += blockDim.x) sh[c] = 0;
  __syncthreads();
}

// every lane of the warp calls this; key < 0 adds nothing
__device__ __forceinline__ void hist_add(int* sh, int key) {
  const unsigned peers = __match_any_sync(0xffffffffu, key);
  if (key >= 0 && __ffs(peers) - 1 == (int)(threadIdx.x & 31)) atomicAdd(&sh[key], __popc(peers));
}

__device__ __forceinline__ void hist_flush(const int* sh, int cells, int64_t* cm) {
  __syncthreads();
  for (int c = threadIdx.x; c < cells; c += blockDim.x) {
    const int v = sh[c];
    if (v) atomicAdd(reinterpret_cast<unsigned long long*>(cm + c), (unsigned long long)v);
  }
}

// histogram cell of (label y, prediction p), or -1 for an ignored or out-of-range label
__device__ __forceinline__ int cell_of(int64_t y, int p, int K, int64_t ignore, int has_ignore, int* status) {
  if (has_ignore && y == ignore) return -1;
  if (y < 0 || y >= K) {
    atomicOr(status, DVA_EVAL_BAD_LABEL);
    return -1;
  }
  return (int)y * K + p;
}

// grid-stride over rows in steps of whole CTAs, so every lane of a warp runs every iteration (hist_add)
template <typename T>
__global__ void __launch_bounds__(kEvThreads)
confusion_scores_kernel(const T* __restrict__ scores, const int64_t* __restrict__ labels,
                        const int* __restrict__ counts, int64_t n, int K, int64_t ignore, int has_ignore,
                        int64_t* __restrict__ cm, int* __restrict__ status) {
  extern __shared__ int sh_hist[];
  hist_zero(sh_hist, K * K);
  for (int64_t base = (int64_t)blockIdx.x * kEvThreads; base < n; base += (int64_t)gridDim.x * kEvThreads) {
    const int64_t i = base + threadIdx.x;
    int key = -1;
    if (i < n && (counts == nullptr || counts[i] != 0)) {
      const int64_t y = labels[i];
      if (!(has_ignore && y == ignore) && y >= 0 && y < K) {
        const T* row = scores + i * K;
        key = (int)y * K + argmax_first(K, [&](int c) { return Cvt<T>::to_f(row[c]); });
      } else {
        key = cell_of(y, 0, K, ignore, has_ignore, status);   // -1, and the status bit of a bad label
      }
    }
    hist_add(sh_hist, key);
  }
  hist_flush(sh_hist, K * K, cm);
}

__global__ void __launch_bounds__(kEvThreads)
confusion_pred_kernel(const int64_t* __restrict__ pred, const int64_t* __restrict__ labels, int64_t n, int K,
                      int64_t ignore, int has_ignore, int64_t* __restrict__ cm, int* __restrict__ status) {
  extern __shared__ int sh_hist[];
  hist_zero(sh_hist, K * K);
  for (int64_t base = (int64_t)blockIdx.x * kEvThreads; base < n; base += (int64_t)gridDim.x * kEvThreads) {
    const int64_t i = base + threadIdx.x;
    int key = -1;
    if (i < n) {
      const int64_t p = pred[i];
      key = cell_of(labels[i], (int)p, K, ignore, has_ignore, status);
      if (key >= 0 && (p < 0 || p >= K)) {
        atomicOr(status, DVA_EVAL_BAD_PRED);
        key = -1;
      }
    }
    hist_add(sh_hist, key);
  }
  hist_flush(sh_hist, K * K, cm);
}

__global__ void __launch_bounds__(kEvThreads)
vote_claim_kernel(const int64_t* __restrict__ ids, int64_t n, int64_t N, int* __restrict__ stamp,
                  int* __restrict__ status) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t id = ids[j];
    if (id < 0 || id >= N) atomicOr(status, DVA_EVAL_BAD_ID);
    else atomicMax(stamp + id, (int)j);
  }
}

// row j is added by the one j that claimed its id, kEvVoteLanes lanes per row (columns strided by kEvVoteLanes); a
// row that lost the claim reads j' != j or the -1 the owner puts back, and adds nothing.  The owner's lanes all
// read the stamp before the __syncwarp after which its first lane puts it back.
constexpr int kEvVoteLanes = 16;

template <typename T>
__global__ void __launch_bounds__(kEvThreads)
vote_add_kernel(const T* __restrict__ outputs, const int64_t* __restrict__ ids, int64_t n, int64_t N, int K,
                float* __restrict__ votes, int* __restrict__ counts, int* __restrict__ stamp) {
  constexpr int kRowsPerWarp = 32 / kEvVoteLanes;
  const int lane = threadIdx.x & 31, sub = lane / kEvVoteLanes, c0 = lane % kEvVoteLanes;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * kRowsPerWarp; base < n; base += warps * kRowsPerWarp) {   // warp-uniform trip count
    const int64_t j = base + sub;
    const int64_t id = j < n ? ids[j] : -1;
    const bool owner = id >= 0 && id < N && stamp[id] == (int)j;
    if (owner) {
      const T* src = outputs + j * K;
      float* dst = votes + id * K;
      for (int c = c0; c < K; c += kEvVoteLanes) dst[c] = __fadd_rn(dst[c], Cvt<T>::to_f(src[c]));
    }
    __syncwarp();
    if (owner && c0 == 0) {
      counts[id] += 1;
      stamp[id] = -1;
    }
  }
}

__global__ void __launch_bounds__(kEvThreads)
nn_vote_kernel(const float* __restrict__ votes, const int* __restrict__ counts, const float* __restrict__ pos,
               int64_t N, int K, const int64_t* __restrict__ voted, int64_t nv, const int64_t* __restrict__ query,
               const int64_t* __restrict__ nbr, int64_t nq, int mode, const int64_t* __restrict__ labels,
               int64_t ignore, int has_ignore, int64_t* __restrict__ pred, int64_t* __restrict__ cm,
               int* __restrict__ status) {
  extern __shared__ int sh_hist[];
  const bool with_cm = labels != nullptr;
  if (with_cm) hist_zero(sh_hist, K * K);
  for (int64_t base = (int64_t)blockIdx.x * kEvThreads; base < nq; base += (int64_t)gridDim.x * kEvThreads) {
    const int64_t q = base + threadIdx.x;
    int key = -1;
    if (q < nq) {
      const int64_t id = query[q];
      bool ok = id >= 0 && id < N;
      int p = 0;
      if (ok && mode == DVA_EVAL_NN_OWN_VOTES && counts[id] > 0) {
        const float* row = votes + id * K;
        p = argmax_first(K, [&](int c) { return row[c]; });
      } else if (ok) {
        const int64_t s = nbr[q];
        const int64_t src = s >= 0 && s < nv ? voted[s] : -1;
        ok = src >= 0 && src < N;
        if (ok) {
          const float dx = __fsub_rn(pos[src * 3 + 0], pos[id * 3 + 0]);
          const float dy = __fsub_rn(pos[src * 3 + 1], pos[id * 3 + 1]);
          const float dz = __fsub_rn(pos[src * 3 + 2], pos[id * 3 + 2]);
          const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
          const float w = __fdiv_rn(1.f, fmaxf(d2, 1e-16f));
          const float cnt = (float)counts[src];
          const bool mean = mode == DVA_EVAL_NN_INTERPOLATE_MEAN;
          const float* row = votes + src * K;
          p = argmax_first(K, [&](int c) {
            const float x = mean ? __fdiv_rn(row[c], cnt) : row[c];
            return __fdiv_rn(__fmul_rn(x, w), w);
          });
        }
      }
      if (!ok) atomicOr(status, DVA_EVAL_BAD_ID);
      pred[q] = p;
      if (ok && with_cm) key = cell_of(labels[id], p, K, ignore, has_ignore, status);
    }
    if (with_cm) hist_add(sh_hist, key);
  }
  if (with_cm) hist_flush(sh_hist, K * K, cm);
}

inline size_t hist_bytes(int K) { return (size_t)K * K * sizeof(int); }

}  // namespace dva_eval

using namespace dva;
using namespace dva_eval;

extern "C" int dva_eval_confusion_scores(const void* scores, int dtype, const int64_t* labels, const int* counts,
                                         int64_t n, int K, int64_t ignore_label, int has_ignore, int64_t* cm,
                                         int* status, void* stream) {
  if (n < 0 || K < 1) return fail(DVA_EINVAL, "eval_confusion_scores: bad sizes");
  if (K > kEvMaxK) return fail(DVA_EUNSUPPORTED, "eval_confusion_scores: K must be in [1, 64]");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "eval_confusion_scores: unknown dtype");
  if (n == 0) return DVA_OK;
  if (!scores || !labels || !cm || !status) return fail(DVA_EINVAL, "eval_confusion_scores: null pointer");
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    confusion_scores_kernel<T><<<grid_cap(n, kEvThreads, 8), kEvThreads, hist_bytes(K), (cudaStream_t)stream>>>(
        (const T*)scores, labels, counts, n, K, ignore_label, has_ignore, cm, status);
  });
  return check_launch("eval_confusion_scores");
}

extern "C" int dva_eval_confusion_pred(const int64_t* pred, const int64_t* labels, int64_t n, int K,
                                       int64_t ignore_label, int has_ignore, int64_t* cm, int* status, void* stream) {
  if (n < 0 || K < 1) return fail(DVA_EINVAL, "eval_confusion_pred: bad sizes");
  if (K > kEvMaxK) return fail(DVA_EUNSUPPORTED, "eval_confusion_pred: K must be in [1, 64]");
  if (n == 0) return DVA_OK;
  if (!pred || !labels || !cm || !status) return fail(DVA_EINVAL, "eval_confusion_pred: null pointer");
  confusion_pred_kernel<<<grid_cap(n, kEvThreads, 8), kEvThreads, hist_bytes(K), (cudaStream_t)stream>>>(
      pred, labels, n, K, ignore_label, has_ignore, cm, status);
  return check_launch("eval_confusion_pred");
}

extern "C" int dva_eval_vote(const void* outputs, int dtype, const int64_t* ids, int64_t n, int64_t N, int K,
                             float* votes, int* counts, int* stamp, int* status, void* stream) {
  if (n < 0 || N < 0 || K < 1) return fail(DVA_EINVAL, "eval_vote: bad sizes");
  if (K > kEvMaxK) return fail(DVA_EUNSUPPORTED, "eval_vote: K must be in [1, 64]");
  if (n > (int64_t)INT32_MAX) return fail(DVA_EUNSUPPORTED, "eval_vote: more than 2^31 - 1 rows");
  if (!known_dtype(dtype)) return fail(DVA_EINVAL, "eval_vote: unknown dtype");
  if (n == 0) return DVA_OK;
  if (!outputs || !ids || !votes || !counts || !stamp || !status) return fail(DVA_EINVAL, "eval_vote: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_cap(n, kEvThreads, 8);
  vote_claim_kernel<<<grid, kEvThreads, 0, st>>>(ids, n, N, stamp, status);
  const int rc = check_launch("eval_vote_claim");
  if (rc != DVA_OK) return rc;
  const int add_grid = grid_cap(n, kEvThreads / kEvVoteLanes, 8);
  with_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    vote_add_kernel<T><<<add_grid, kEvThreads, 0, st>>>((const T*)outputs, ids, n, N, K, votes, counts, stamp);
  });
  return check_launch("eval_vote_add");
}

extern "C" int dva_eval_nn_vote(const float* votes, const int* counts, const float* pos, int64_t N, int K,
                                const int64_t* voted, int64_t nv, const int64_t* query, const int64_t* nbr, int64_t nq,
                                int mode, const int64_t* labels, int64_t ignore_label, int has_ignore, int64_t* pred,
                                int64_t* cm, int* status, void* stream) {
  if (N < 0 || nv < 0 || nq < 0 || K < 1) return fail(DVA_EINVAL, "eval_nn_vote: bad sizes");
  if (K > kEvMaxK) return fail(DVA_EUNSUPPORTED, "eval_nn_vote: K must be in [1, 64]");
  if (mode != DVA_EVAL_NN_INTERPOLATE && mode != DVA_EVAL_NN_INTERPOLATE_MEAN && mode != DVA_EVAL_NN_OWN_VOTES)
    return fail(DVA_EINVAL, "eval_nn_vote: unknown mode");
  if (nq == 0) return DVA_OK;
  if (nv == 0) return fail(DVA_EINVAL, "eval_nn_vote: empty search set");
  if (!votes || !counts || !pos || !voted || !query || !nbr || !pred || !status || (labels && !cm))
    return fail(DVA_EINVAL, "eval_nn_vote: null pointer");
  nn_vote_kernel<<<grid_cap(nq, kEvThreads, 8), kEvThreads, labels ? hist_bytes(K) : 0, (cudaStream_t)stream>>>(
      votes, counts, pos, N, K, voted, nv, query, nbr, nq, mode, labels, ignore_label, has_ignore, pred, cm, status);
  return check_launch("eval_nn_vote");
}
