// CSR bookkeeping kernels (integer, bit-exact): pointers from sorted dense ids with empty
// groups inserted (csr.py:158-172 + :197-229, used by ImageMapping.from_dense image.py:1787-1793)
// and the value index of a group selection (csr.py:235-264, CSRData.__getitem__).
// The reference builds these with chains of where/cat/cumsum/repeat_interleave/arange, each a
// launch plus a temporary; here each is one pass: 8 B read + 8 B written per element.
#include "dva_common.cuh"

namespace dva {

// boundary j (0..n): groups (ids[j-1], ids[j]] start at item j.  Every ptr slot is written once.
__global__ void __launch_bounds__(256)
csr_pointers_kernel(const int64_t* __restrict__ ids, int64_t* __restrict__ ptr, int64_t n,
                    int64_t num_groups) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j <= n;
       j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t prev = (j == 0) ? -1 : ids[j - 1];
    const int64_t cur = (j == n) ? num_groups : ids[j];
    for (int64_t g = prev + 1; g <= cur && g <= num_groups; ++g) ptr[g] = j;
  }
}

__global__ void __launch_bounds__(256)
csr_select_values_kernel(const int64_t* __restrict__ ptr, const int64_t* __restrict__ sel,
                         const int64_t* __restrict__ ptr_new, int64_t* __restrict__ val_idx,
                         int64_t k) {
  // 8 lanes per selected group
  const int sub = threadIdx.x & 7;
  const int64_t groups = ((int64_t)gridDim.x * blockDim.x) >> 3;
  for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 3; i < k; i += groups) {
    const int64_t src0 = ptr[sel[i]], d0 = ptr_new[i], d1 = ptr_new[i + 1];
    for (int64_t p = d0 + sub; p < d1; p += 8) val_idx[p] = src0 + (p - d0);
  }
}

}  // namespace dva

using namespace dva;

extern "C" int dva_csr_pointers_from_sorted(const int64_t* ids, int64_t* ptr, int64_t n,
                                            int64_t num_groups, void* stream) {
  if (n < 0 || num_groups < 0) return fail(DVA_EINVAL, "csr_pointers_from_sorted: negative size");
  if (!ptr || (n > 0 && !ids)) return fail(DVA_EINVAL, "csr_pointers_from_sorted: null pointer");
  csr_pointers_kernel<<<grid_cap(n + 1, 256, 16), 256, 0, (cudaStream_t)stream>>>(ids, ptr, n, num_groups);
  return check_launch("csr_pointers");
}

extern "C" int dva_csr_select_values(const int64_t* ptr, const int64_t* sel,
                                     const int64_t* ptr_new, int64_t* val_idx, int64_t k,
                                     int64_t n_new_items, void* stream) {
  if (k < 0 || n_new_items < 0) return fail(DVA_EINVAL, "csr_select_values: negative size");
  if (k == 0 || n_new_items == 0) return DVA_OK;
  if (!ptr || !sel || !ptr_new || !val_idx) return fail(DVA_EINVAL, "csr_select_values: null pointer");
  csr_select_values_kernel<<<grid_cap(k * 8, 256, 16), 256, 0, (cudaStream_t)stream>>>(ptr, sel, ptr_new, val_idx, k);
  return check_launch("csr_select_values");
}
