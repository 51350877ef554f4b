"""Kernel table of libdva_resnet.so, the ADE20K ResNet-18 encoder (namespace dva_resnet::, csrc/resnet.cu).

tests/test_gpu_library_matrix.py runs every instantiation on the GPU under the kernel recorder and asserts, by name,
that it ran; tests/test_library_tables.py checks the table against the library without a GPU.  This file checks
that an argument error of the library is reported through _lib.last_error() without a launch.
rn_conv_gemm_kernel<MODE>: 0 = forward, 1 = data gradient."""
from deepviewagg_b200 import _lib
import test_kernel_matrix_table as KM
from test_kernel_matrix_table import kname

NAMESPACE = "dva_resnet::"
FAMILIES = ("rn_conv_gemm_kernel", "rn_conv_wgrad_kernel", "rn_wgrad_reduce_kernel", "rn_weight_prep_kernel",
            "rn_bn_stats_kernel", "rn_bn_apply_kernel", "rn_bn_bwd_partial_kernel", "rn_bn_bwd_reduce_kernel",
            "rn_bn_bwd_dz_kernel", "rn_maxpool_kernel", "rn_maxpool_bwd_kernel", "rn_resize_kernel",
            "rn_resize_bwd_kernel")


def canonical(name):
    return KM.canonical(name, FAMILIES, NAMESPACE)


# every kernel runs in the one scenario of tests/test_gpu_library_matrix.py: a Pyramid train step (forward and
# backward, with the input's gradient)
TABLE = {kname("rn_conv_gemm_kernel", m): "pyramid" for m in range(2)}
TABLE.update({f: "pyramid" for f in FAMILIES[1:]})


def test_errors_reach_the_shared_error_string():
    lib = _lib.load_resnet()
    n0 = _lib.launch_count()
    rc = lib.dva_resnet_conv_bn_fwd(None, 1, 8, 8, 3, None, 64, 3, 2, 2, 1, 1e-3, 1e-5, None, None, None, None, None,
                                    None, 0, None)
    assert rc == _lib.DVA_EINVAL and "unsupported shape (T 3, stride 2, dilation 2)" in _lib.last_error()
    rc = lib.dva_resnet_conv_dgrad(None, 1, 8, 8, 4, 8, None, 1, 1, 1, None, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_conv_dgrad: null pointer"
    rc = lib.dva_resnet_conv_wgrad(None, None, 0, 8, 8, 4, 8, 3, 1, 4, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_conv_wgrad: bad sizes"
    rc = lib.dva_resnet_resize(None, 1, 4, 4, 8, 8, 8, 0.5, 0.5, None, 8, 4, None)
    assert rc == _lib.DVA_EINVAL and "column slice" in _lib.last_error()
    rc = lib.dva_resnet_maxpool(None, 1, 0, 4, 8, None, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "resnet_maxpool: bad sizes"
    assert _lib.launch_count() == n0
    assert lib.dva_resnet_wgrad_workspace_bytes(1, 8, 8, 4, 8, 2, 1, 1) == 0
    assert lib.dva_resnet_fwd_workspace_bytes(1, 8, 8, 8) > 0


def test_canonical_names():
    assert canonical("void dva_resnet::rn_conv_gemm_kernel<1>(dva_resnet::ConvArgs)") == "rn_conv_gemm_kernel<1>"
    assert canonical("dva_resnet::rn_maxpool_kernel(float const*)") == "rn_maxpool_kernel"
    assert canonical("void dva_unet::convt_gemm_kernel<3>(dva_unet::ConvTArgs)") is None
