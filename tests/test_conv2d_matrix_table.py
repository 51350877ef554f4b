"""Kernel table of libdva_conv2d.so, the image encoder's convolutions and GroupNorm (namespace dva_conv2d::,
csrc/conv2d.cu).

tests/test_gpu_library_matrix.py runs every instantiation on the GPU under the kernel recorder and asserts, by name,
that it ran; tests/test_library_tables.py checks the table against the library without a GPU.  This file checks
that an argument error of the library is reported through _lib.last_error() (the libraries share the error
string).
conv_gemm_kernel<MODE>: 0/1/2 = forward 3x3 reflect / 2x2 stride 2 / 1x1, 3/4/5 = data gradient of the same;
conv_wgrad_kernel<KIND>: KIND = DVA_CONV_3X3_REFLECT (0), DVA_CONV_2X2_S2 (1), DVA_CONV_1X1 (2)."""
from deepviewagg_b200 import _lib
import test_kernel_matrix_table as KM
from test_kernel_matrix_table import kname

NAMESPACE = "dva_conv2d::"
FAMILIES = ("conv_gemm_kernel", "conv_wgrad_kernel", "gn_stats_kernel", "wgrad_reduce_kernel", "weight_prep_kernel",
            "weight_prep_bwd_kernel", "gn_apply_kernel", "gn_bwd_partial_kernel", "gn_bwd_sums_kernel",
            "gn_bwd_coef_kernel", "gn_bwd_dz_kernel")


def canonical(name):
    return KM.canonical(name, FAMILIES, NAMESPACE)


# every kernel runs in the one scenario of tests/test_gpu_library_matrix.py: forward + backward of a two-stage
# encoder (3x3 conv_in, then a 2x2 conv_in and two ResBlocks, the first with a 1x1 downsample) with the input's
# gradient
TABLE = {kname("conv_gemm_kernel", m): "encoder" for m in range(6)}
TABLE.update({kname("conv_wgrad_kernel", k): "encoder" for k in range(3)})
TABLE.update({f: "encoder" for f in FAMILIES[2:]})


def test_errors_reach_the_shared_error_string():
    lib = _lib.load_conv()
    n0 = _lib.launch_count()
    rc = lib.dva_conv2d_fwd(None, 1, 1, 8, 4, None, None, 8, 0, 1, 1e-5, None, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error().startswith("conv2d_fwd:") and ">= 2" in _lib.last_error()
    rc = lib.dva_conv2d_fwd(None, 1, 8, 8, 4, None, None, 8, 7, 1, 1e-5, None, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and "unknown kind" in _lib.last_error()
    rc = lib.dva_conv2d_fwd(None, 1, 8, 8, 4, None, None, 24, 0, 5, 1e-5, None, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and "groups must divide" in _lib.last_error()
    rc = lib.dva_conv2d_gn_bwd(None, None, 1, 4, 8, 3, None, None, None, None, 0.0, None, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error().startswith("conv2d_gn_bwd:")
    rc = lib.dva_conv2d_dgrad(None, 1, 8, 8, 4, 8, None, 1, None, None, None)
    assert rc == _lib.DVA_EINVAL and "null pointer" in _lib.last_error()
    assert _lib.launch_count() == n0
    assert lib.dva_conv2d_wgrad_workspace_bytes(1, 1, 8, 4, 8, 0) == 0


def test_canonical_names():
    assert canonical("void dva_conv2d::conv_gemm_kernel<3>(dva_conv2d::GemmArgs)") == "conv_gemm_kernel<3>"
    assert canonical("dva_conv2d::gn_apply_kernel(float const*)") == "gn_apply_kernel"
    assert canonical("void dva::csr_nll_fwd_kernel<float>(float const*)") is None
