"""Kernel table of libdva_resnet.so, the ADE20K ResNet-18 encoder (namespace dva_resnet::, csrc/resnet.cu).

tests/test_gpu_resnet18_matrix.py runs every instantiation on the GPU under the kernel recorder and asserts, by name,
that it ran.  This file checks, without a GPU, that
  * the table holds exactly the kernels compiled into libdva_resnet.so, all of them in dva_resnet::;
  * no kernel family of libdva_resnet.so appears in libdva_b200.so, libdva_eval.so, libdva_conv2d.so or
    libdva_unet.so;
  * include/dva_resnet.h, _lib.RESNET_SIGNATURES and the exported symbols agree, and are disjoint from the other
    tables of signatures;
  * an argument error of the new library is reported through _lib.last_error() without a launch.
rn_conv_gemm_kernel<MODE>: 0 = forward, 1 = data gradient."""
import os

import pytest

from deepviewagg_b200 import _lib
from test_conv2d_matrix_table import _declared
from test_kernel_matrix_table import kname, parse_kernel
from test_loss_matrix_table import demangled_kernels

NAMESPACE = "dva_resnet::"
FAMILIES = ("rn_conv_gemm_kernel", "rn_conv_wgrad_kernel", "rn_wgrad_reduce_kernel", "rn_weight_prep_kernel",
            "rn_bn_stats_kernel", "rn_bn_apply_kernel", "rn_bn_bwd_partial_kernel", "rn_bn_bwd_reduce_kernel",
            "rn_bn_bwd_dz_kernel", "rn_maxpool_kernel", "rn_maxpool_bwd_kernel", "rn_resize_kernel",
            "rn_resize_bwd_kernel")


def canonical(name):
    """Demangled dva_resnet:: kernel name -> 'family<args>'; None for anything else."""
    s = name.strip()
    if s.startswith("void "):
        s = s[5:]
    if not s.startswith(NAMESPACE):
        return None
    p = parse_kernel("dva::" + s[len(NAMESPACE):])
    if p is None or p[0] not in FAMILIES:
        return None
    return kname(p[0], *p[1])


# every kernel runs in the one scenario of tests/test_gpu_resnet18_matrix.py: a Pyramid train step (forward and
# backward, with the input's gradient)
TABLE = {kname("rn_conv_gemm_kernel", m): "pyramid" for m in range(2)}
TABLE.update({f: "pyramid" for f in FAMILIES[1:]})


def _built():
    for p in (_lib.LIB_PATH, _lib.RESNET_LIB_PATH):
        if not os.path.exists(p):
            pytest.fail(f"{p} is not built")
    return _lib.RESNET_LIB_PATH


def test_table_matches_library():
    names = [n for n in demangled_kernels(_built()) if "__internal" not in n]
    outside = sorted(n for n in names if not n.replace("void ", "", 1).startswith(NAMESPACE))
    assert not outside, outside
    built = {canonical(n) for n in names}
    assert None not in built, names
    assert built == set(TABLE), {"compiled without a case": sorted(built - set(TABLE)),
                                 "case without a kernel": sorted(set(TABLE) - built)}
    assert len(TABLE) == 14


def test_no_kernel_family_shared_with_the_other_libraries():
    _built()
    ours = {canonical(n).split("<")[0] for n in demangled_kernels(_lib.RESNET_LIB_PATH) if canonical(n)}
    assert ours == set(FAMILIES)
    for other in (_lib.LIB_PATH, _lib.EVAL_LIB_PATH, _lib.CONV_LIB_PATH, _lib.UNET_LIB_PATH):
        names = {n.replace("void ", "", 1).split("(")[0] for n in demangled_kernels(other)}
        assert not any(n.startswith(NAMESPACE) for n in names)
        assert not {n for n in names if n.split("::")[-1].split("<")[0] in ours}


def test_header_signatures_and_exports_agree():
    _built()
    names = _declared("dva_resnet.h")
    assert names == set(_lib.RESNET_SIGNATURES)
    assert all(n.startswith("dva_resnet_") for n in names)
    for other in (_lib.SIGNATURES, _lib.EVAL_SIGNATURES, _lib.CONV_SIGNATURES, _lib.UNET_SIGNATURES):
        assert not names & set(other)
    lib = _lib.load_resnet()
    for n in names:
        assert hasattr(lib, n), n
        assert _lib.entry(n) is getattr(lib, n)
    assert _lib.entry("dva_unet_fwd") is getattr(_lib.load_unet(), "dva_unet_fwd")


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
