"""deepviewagg_b200 -- H100 (sm_90a) implementation of DeepViewAgg's multi-view aggregation
hot path behind the reference's torch_points3d/modules/multimodal operator API.

Layout (only what the path needs):
  csrc/                 hand-written CUDA kernels + the C ABI (include/dva_b200.h)
  _lib.py               ctypes binding of libdva_b200.so (no CPU fallback)
  ops.py                autograd operators over the C ABI
  modules/multimodal/   drop-in mirror of torch_points3d/modules/multimodal/{pooling,fusion,modules}.py
  core/multimodal/      CSR / ImageMapping index structures (csr.py, image.py) and visibility
  core/common_modules.py MLP / FastBatchNorm1d with the reference's parameter names
  utils/multimodal.py   lexicographic sort/unique helpers
  install.py            registers the mirror under the reference's module paths (drop-in)
"""
__version__ = "0.1.0"
