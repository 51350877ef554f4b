"""Kernel table of libdva_unet.so, the image decoder's transposed convolutions (namespace dva_unet::,
csrc/conv2d_up.cu).

tests/test_gpu_library_matrix.py runs every instantiation on the GPU under the kernel recorder and asserts, by name,
that it ran; tests/test_library_tables.py checks the table against the library without a GPU.  This file checks
that an argument error of the library is reported through _lib.last_error() without a launch.
convt_gemm_kernel<MODE>: 0 = 2x2 stride-2 upsampling forward, 1 = 3x3 transposed forward, 2 = its data gradient,
3 = the upsampling's data gradient; convt_wgrad_kernel<KIND>: KIND = DVA_UNET_UP_2X2 (0), DVA_UNET_T_3X3 (1)."""
from deepviewagg_b200 import _lib
import test_kernel_matrix_table as KM
from test_kernel_matrix_table import kname

NAMESPACE = "dva_unet::"
FAMILIES = ("convt_gemm_kernel", "convt_wgrad_kernel", "convt_stats_kernel", "convt_wgrad_reduce_kernel",
            "convt_weight_prep_kernel", "convt_weight_prep_bwd_kernel", "unary_act_kernel", "unary_act_bwd_kernel")


def canonical(name):
    return KM.canonical(name, FAMILIES, NAMESPACE)


# every kernel runs in the one scenario of tests/test_gpu_library_matrix.py: forward + backward of a small UNet (2x2
# upsampling stages, transposed 3x3 blocks) and a ReLUWS last_conv, with the input's gradient
TABLE = {kname("convt_gemm_kernel", m): "unet" for m in range(4)}
TABLE.update({kname("convt_wgrad_kernel", k): "unet" for k in range(2)})
TABLE.update({f: "unet" for f in FAMILIES[2:]})


def test_errors_reach_the_shared_error_string():
    lib = _lib.load_unet()
    n0 = _lib.launch_count()
    rc = lib.dva_unet_fwd(None, 1, 8, 8, 4, None, None, 8, 5, 1, 1e-5, None, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "unet_fwd: unknown kind"
    rc = lib.dva_unet_fwd(None, 1, 8, 8, 4, None, None, 24, 0, 5, 1e-5, None, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and "groups must divide" in _lib.last_error()
    rc = lib.dva_unet_fwd(None, 1, 8, 8, 4, None, None, 4096, 1, 256, 1e-5, None, None, None, None, 0, None)
    assert rc == _lib.DVA_EUNSUPPORTED and "at most 128 groups" in _lib.last_error()
    rc = lib.dva_unet_dgrad(None, 1, 8, 8, 4, 8, None, 1, None, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "unet_dgrad: null pointer"
    rc = lib.dva_unet_wgrad(None, None, 0, 8, 8, 4, 8, 0, None, None, None, 0, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error() == "unet_wgrad: bad sizes"
    rc = lib.dva_unet_act(None, 16, 0.0, None, None)
    assert rc == _lib.DVA_EINVAL and _lib.last_error().startswith("unet_act:")
    assert _lib.launch_count() == n0
    assert lib.dva_unet_wgrad_workspace_bytes(1, 8, 8, 4, 8, 3) == 0
    assert lib.dva_unet_fwd_workspace_bytes(1, 8, 8, 8, 1, 0) > 0


def test_canonical_names():
    assert canonical("void dva_unet::convt_gemm_kernel<3>(dva_unet::ConvTArgs)") == "convt_gemm_kernel<3>"
    assert canonical("dva_unet::unary_act_kernel(float const*)") == "unary_act_kernel"
    assert canonical("void dva_conv2d::conv_gemm_kernel<3>(dva_conv2d::GemmArgs)") is None
