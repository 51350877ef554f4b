"""Kernel table of libdva_eval.so, the segmentation evaluation kernels (namespace dva_eval::, csrc/eval_metrics.cu).

tests/test_gpu_eval_matrix.py runs every instantiation on the GPU under the kernel recorder and asserts, by name,
that it ran; tests/test_library_tables.py checks the table against the library without a GPU.  This file checks
that an argument error of the library is reported through _lib.last_error() (the libraries share the error
string), and that the operators refuse CPU tensors.
Every result of these kernels is an integer or an exact fp32 sequence, so the GPU matrix compares bits."""
import pytest

from deepviewagg_b200 import _lib
import test_kernel_matrix_table as KM
from test_kernel_matrix_table import CPP, DTYPES, kname

NAMESPACE = "dva_eval::"
FAMILIES = ("confusion_scores_kernel", "confusion_pred_kernel", "vote_claim_kernel", "vote_add_kernel",
            "nn_vote_kernel")


def canonical(name):
    return KM.canonical(name, FAMILIES, NAMESPACE)


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
