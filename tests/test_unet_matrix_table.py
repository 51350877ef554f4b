"""Kernel table of libdva_unet.so, the image decoder's transposed convolutions (namespace dva_unet::,
csrc/conv2d_up.cu).

tests/test_gpu_unet_matrix.py runs every instantiation on the GPU under the kernel recorder and asserts, by name,
that it ran.  This file checks, without a GPU, that
  * the table holds exactly the kernels compiled into libdva_unet.so, all of them in dva_unet::;
  * no kernel family of libdva_unet.so appears in libdva_b200.so, libdva_eval.so or libdva_conv2d.so;
  * include/dva_unet.h, _lib.UNET_SIGNATURES and the exported symbols agree, and are disjoint from the other three
    tables of signatures;
  * an argument error of the new library is reported through _lib.last_error() without a launch.
convt_gemm_kernel<MODE>: 0 = 2x2 stride-2 upsampling forward, 1 = 3x3 transposed forward, 2 = its data gradient,
3 = the upsampling's data gradient; convt_wgrad_kernel<KIND>: KIND = DVA_UNET_UP_2X2 (0), DVA_UNET_T_3X3 (1)."""
import pytest

from deepviewagg_b200 import _lib
from test_conv2d_matrix_table import _declared
from test_kernel_matrix_table import kname, parse_kernel
from test_loss_matrix_table import demangled_kernels

NAMESPACE = "dva_unet::"
FAMILIES = ("convt_gemm_kernel", "convt_wgrad_kernel", "convt_stats_kernel", "convt_wgrad_reduce_kernel",
            "convt_weight_prep_kernel", "convt_weight_prep_bwd_kernel", "unary_act_kernel", "unary_act_bwd_kernel")


def canonical(name):
    """Demangled dva_unet:: kernel name -> 'family<args>'; None for anything else."""
    s = name.strip()
    if s.startswith("void "):
        s = s[5:]
    if not s.startswith(NAMESPACE):
        return None
    p = parse_kernel("dva::" + s[len(NAMESPACE):])
    if p is None or p[0] not in FAMILIES:
        return None
    return kname(p[0], *p[1])


# every kernel runs in the one scenario of tests/test_gpu_unet_matrix.py: forward + backward of a small UNet (2x2
# upsampling stages, transposed 3x3 blocks) and a ReLUWS last_conv, with the input's gradient
TABLE = {kname("convt_gemm_kernel", m): "unet" for m in range(4)}
TABLE.update({kname("convt_wgrad_kernel", k): "unet" for k in range(2)})
TABLE.update({f: "unet" for f in FAMILIES[2:]})


def _built():
    import os
    for p in (_lib.LIB_PATH, _lib.UNET_LIB_PATH):
        if not os.path.exists(p):
            pytest.fail(f"{p} is not built")
    return _lib.UNET_LIB_PATH


def test_table_matches_library():
    names = [n for n in demangled_kernels(_built()) if "__internal" not in n]
    outside = sorted(n for n in names if not n.replace("void ", "", 1).startswith(NAMESPACE))
    assert not outside, outside
    built = {canonical(n) for n in names}
    assert None not in built, names
    assert built == set(TABLE), {"compiled without a case": sorted(built - set(TABLE)),
                                 "case without a kernel": sorted(set(TABLE) - built)}
    assert len(TABLE) == 12


def test_no_kernel_family_shared_with_the_other_libraries():
    _built()
    ours = {canonical(n).split("<")[0] for n in demangled_kernels(_lib.UNET_LIB_PATH) if canonical(n)}
    assert ours == set(FAMILIES)
    for other in (_lib.LIB_PATH, _lib.EVAL_LIB_PATH, _lib.CONV_LIB_PATH):
        names = {n.replace("void ", "", 1).split("(")[0] for n in demangled_kernels(other)}
        assert not any(n.startswith(NAMESPACE) for n in names)
        assert not {n for n in names if n.split("::")[-1].split("<")[0] in ours}


def test_header_signatures_and_exports_agree():
    _built()
    names = _declared("dva_unet.h")
    assert names == set(_lib.UNET_SIGNATURES)
    assert all(n.startswith("dva_unet_") for n in names)
    for other in (_lib.SIGNATURES, _lib.EVAL_SIGNATURES, _lib.CONV_SIGNATURES):
        assert not names & set(other)
    lib = _lib.load_unet()
    for n in names:
        assert hasattr(lib, n), n
        assert _lib.entry(n) is getattr(lib, n)
    assert _lib.entry("dva_conv2d_fwd") is getattr(_lib.load_conv(), "dva_conv2d_fwd")


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
