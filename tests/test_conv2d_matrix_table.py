"""Kernel table of libdva_conv2d.so, the image encoder's convolutions and GroupNorm (namespace dva_conv2d::,
csrc/conv2d.cu).

tests/test_gpu_conv2d_matrix.py runs every instantiation on the GPU under the kernel recorder and asserts, by name,
that it ran.  This file checks, without a GPU, that
  * the table holds exactly the kernels compiled into libdva_conv2d.so, all of them in dva_conv2d::;
  * no kernel name of libdva_conv2d.so appears in libdva_b200.so or libdva_eval.so;
  * include/dva_conv2d.h, _lib.CONV_SIGNATURES and the exported symbols agree, and are disjoint from the other
    two tables of signatures;
  * an argument error of the new library is reported through _lib.last_error() (the libraries share the error
    string).
conv_gemm_kernel<MODE>: 0/1/2 = forward 3x3 reflect / 2x2 stride 2 / 1x1, 3/4/5 = data gradient of the same;
conv_wgrad_kernel<KIND>: KIND = DVA_CONV_3X3_REFLECT (0), DVA_CONV_2X2_S2 (1), DVA_CONV_1X1 (2)."""
import os
import re

import pytest

from conftest import ROOT
from deepviewagg_b200 import _lib
from test_kernel_matrix_table import kname, parse_kernel
from test_loss_matrix_table import demangled_kernels

NAMESPACE = "dva_conv2d::"
FAMILIES = ("conv_gemm_kernel", "conv_wgrad_kernel", "gn_stats_kernel", "wgrad_reduce_kernel", "weight_prep_kernel",
            "weight_prep_bwd_kernel", "gn_apply_kernel", "gn_bwd_partial_kernel", "gn_bwd_sums_kernel",
            "gn_bwd_coef_kernel", "gn_bwd_dz_kernel")


def canonical(name):
    """Demangled dva_conv2d:: kernel name -> 'family<args>'; None for anything else."""
    s = name.strip()
    if s.startswith("void "):
        s = s[5:]
    if not s.startswith(NAMESPACE):
        return None
    p = parse_kernel("dva::" + s[len(NAMESPACE):])
    if p is None or p[0] not in FAMILIES:
        return None
    return kname(p[0], *p[1])


# every kernel runs in the one scenario of tests/test_gpu_conv2d_matrix.py: forward + backward of a two-stage
# encoder (3x3 conv_in, then a 2x2 conv_in and two ResBlocks, the first with a 1x1 downsample) with the input's
# gradient
TABLE = {kname("conv_gemm_kernel", m): "encoder" for m in range(6)}
TABLE.update({kname("conv_wgrad_kernel", k): "encoder" for k in range(3)})
TABLE.update({f: "encoder" for f in FAMILIES[2:]})


def _built():
    for p in (_lib.LIB_PATH, _lib.CONV_LIB_PATH):
        if not os.path.exists(p):
            pytest.fail(f"{p} is not built")
    return _lib.CONV_LIB_PATH


def test_table_matches_library():
    names = demangled_kernels(_built())
    names = [n for n in names if "__internal" not in n]
    outside = sorted(n for n in names if not n.replace("void ", "", 1).startswith(NAMESPACE))
    assert not outside, outside
    built = {canonical(n) for n in names}
    assert None not in built, names
    assert built == set(TABLE), {"compiled without a case": sorted(built - set(TABLE)),
                                 "case without a kernel": sorted(set(TABLE) - built)}
    assert len(TABLE) == 18


def test_no_kernel_name_shared_with_the_other_libraries():
    _built()
    ours = {canonical(n).split("<")[0] for n in demangled_kernels(_lib.CONV_LIB_PATH) if canonical(n)}
    for other in (_lib.LIB_PATH, _lib.EVAL_LIB_PATH):
        names = {n.replace("void ", "", 1).split("(")[0] for n in demangled_kernels(other)}
        assert not any(n.startswith(NAMESPACE) for n in names)
        assert not {n for n in names if n.split("::")[-1].split("<")[0] in ours}


def _declared(header):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(re.findall(r"\b(dva_[a-z0-9_]+)\s*\(", text))


def test_header_signatures_and_exports_agree():
    _built()
    names = _declared("dva_conv2d.h")
    assert names == set(_lib.CONV_SIGNATURES)
    assert all(n.startswith("dva_conv2d_") for n in names)
    assert not names & set(_lib.SIGNATURES) and not names & set(_lib.EVAL_SIGNATURES)
    lib = _lib.load_conv()
    for n in names:
        assert hasattr(lib, n), n
        assert _lib.entry(n) is getattr(lib, n)
    assert _lib.entry("dva_knn_query") is getattr(_lib.load(), "dva_knn_query")
    assert _lib.entry("dva_eval_vote") is getattr(_lib.load_eval(), "dva_eval_vote")


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
