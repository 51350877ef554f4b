"""Kernel table of libdva_eval.so, the segmentation evaluation kernels (namespace dva_eval::, csrc/eval_metrics.cu).

tests/test_gpu_eval_matrix.py runs every instantiation on the GPU under the kernel recorder and asserts, by name,
that it ran.  This file checks, without a GPU, that
  * the table holds exactly the kernels compiled into libdva_eval.so, all of them in dva_eval::;
  * no kernel name of libdva_eval.so appears in libdva_b200.so;
  * include/dva_eval.h, _lib.EVAL_SIGNATURES and the exported symbols agree, and the two tables of signatures
    are disjoint;
  * an argument error of the new library is reported through _lib.last_error() (the libraries share the
    error string).
Every result of these kernels is an integer or an exact fp32 sequence, so the GPU matrix compares bits."""
import os
import re

import pytest

from conftest import ROOT
from deepviewagg_b200 import _lib
from test_kernel_matrix_table import CPP, DTYPES, kname, parse_kernel
from test_loss_matrix_table import demangled_kernels

NAMESPACE = "dva_eval::"
FAMILIES = ("confusion_scores_kernel", "confusion_pred_kernel", "vote_claim_kernel", "vote_add_kernel",
            "nn_vote_kernel")


def canonical(name):
    """Demangled dva_eval:: kernel name -> 'family<args>'; None for anything else."""
    s = name.strip()
    if s.startswith("void "):
        s = s[5:]
    if not s.startswith(NAMESPACE):
        return None
    p = parse_kernel("dva::" + s[len(NAMESPACE):])
    if p is None or p[0] not in FAMILIES:
        return None
    return kname(p[0], *p[1])


def _cases():
    c = {}
    for dt in DTYPES:
        c[kname("confusion_scores_kernel", CPP[dt])] = f"scores_{dt}"
        c[kname("vote_add_kernel", CPP[dt])] = f"vote_{dt}"
    c["confusion_pred_kernel"] = "pred"
    c["vote_claim_kernel"] = "vote_f32"
    c["nn_vote_kernel"] = "nn"
    return c


TABLE = _cases()


def _built():
    for p in (_lib.LIB_PATH, _lib.EVAL_LIB_PATH):
        if not os.path.exists(p):
            pytest.fail(f"{p} is not built")
    return _lib.EVAL_LIB_PATH


def test_table_matches_library():
    names = demangled_kernels(_built())
    names = [n for n in names if "__internal" not in n]    # libdevice's static slow paths, not kernels of ours
    outside = sorted(n for n in names if not n.replace("void ", "", 1).startswith(NAMESPACE))
    assert not outside, outside
    built = {canonical(n) for n in names}
    assert None not in built, names
    assert built == set(TABLE), {"compiled without a case": sorted(built - set(TABLE)),
                                 "case without a kernel": sorted(set(TABLE) - built)}
    assert len(TABLE) == 9


def test_no_eval_kernel_in_the_first_library():
    _built()
    first = {n.replace("void ", "", 1).split("(")[0] for n in demangled_kernels(_lib.LIB_PATH)}
    assert not any(n.startswith(NAMESPACE) for n in first)
    bare = {canonical(n).split("<")[0] for n in demangled_kernels(_lib.EVAL_LIB_PATH) if canonical(n)}
    assert not {n for n in first if n.split("::")[-1].split("<")[0] in bare}


def _declared(header):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(re.findall(r"\b(dva_[a-z0-9_]+)\s*\(", text))


def test_header_signatures_and_exports_agree():
    _built()
    names = _declared("dva_eval.h")
    assert names == set(_lib.EVAL_SIGNATURES)
    assert all(n.startswith("dva_eval_") for n in names)
    assert not names & set(_lib.SIGNATURES)
    lib = _lib.load_eval()
    for n in names:
        assert hasattr(lib, n), n
        assert _lib.entry(n) is getattr(lib, n)
    assert _lib.entry("dva_knn_query") is getattr(_lib.load(), "dva_knn_query")


def test_errors_reach_the_shared_error_string():
    lib = _lib.load_eval()
    rc = lib.dva_eval_confusion_scores(None, 0, None, None, 10, 65, 0, 0, None, None, None)
    assert rc == _lib.DVA_EUNSUPPORTED and _lib.last_error().startswith("eval_confusion_scores:")
    rc = lib.dva_eval_vote(None, 7, None, 4, 4, 4, None, None, None, None, None)
    assert rc == _lib.DVA_EINVAL and "unknown dtype" in _lib.last_error()
    rc = lib.dva_eval_nn_vote(None, None, None, 10, 13, None, 0, None, None, 4, 0, None, 0, 0, None, None, None, None)
    assert rc == _lib.DVA_EINVAL and "empty search set" in _lib.last_error()
    rc = lib.dva_eval_nn_vote(None, None, None, 10, 13, None, 1, None, None, 4, 3, None, 0, 0, None, None, None, None)
    assert rc == _lib.DVA_EINVAL and "unknown mode" in _lib.last_error()
    # nothing to do is not an error, and launches nothing
    n0 = _lib.launch_count()
    assert lib.dva_eval_confusion_pred(None, None, 0, 13, 0, 0, None, None, None) == 0
    assert _lib.launch_count() == n0


def test_ops_reject_cpu_tensors():
    import torch
    from deepviewagg_b200 import ops
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        ops.confusion_update(torch.zeros(3, 3, dtype=torch.int64), torch.zeros(4, 3), torch.zeros(4, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        ops.vote(torch.zeros(4, 3), torch.zeros(4, dtype=torch.int32), torch.zeros(4, dtype=torch.int32),
                 torch.zeros(2, dtype=torch.int64), torch.zeros(2, 3))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        ops.full_res_predict(torch.zeros(4, 3), torch.zeros(4, dtype=torch.int32), torch.zeros(4, 3))


def test_canonical_names():
    assert canonical("void dva_eval::confusion_scores_kernel<__half>(__half const*, long const*, int const*, long, "
                     "int, long, int, long*, int*)") == "confusion_scores_kernel<__half>"
    assert canonical("dva_eval::nn_vote_kernel(float const*)") == "nn_vote_kernel"
    assert canonical("void dva::csr_nll_fwd_kernel<float>(float const*)") is None
