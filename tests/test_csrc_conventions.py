"""The launch convention of the C++ launchers: every host-side decision shared by the kernel files (dtype, reduce
and lane dispatch, grid sizing, workspace alignment) lives once, in csrc/dva_common.cuh; the launchers call it.
And the one hazard of that convention: with_dtype maps any code it does not know to __half, so every entry point
has to reject an unknown dtype or reduce code itself before it dispatches."""
import os
import re

import pytest
import torch

from conftest import ROOT
from deepviewagg_b200 import _lib

CSRC = os.path.join(ROOT, "deepviewagg_b200", "csrc")
COMMON = "dva_common.cuh"


def _sources():
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h")):
            yield f, open(os.path.join(CSRC, f)).read()


def _find(pattern):
    return [f"{f}: {m.group(0).strip()}" for f, src in _sources() for m in re.finditer(pattern, src, re.M)]


def test_no_function_like_macros():
    """Launch and dispatch code is written as C++ (templates, lambdas), not macros; tuning values may stay
    `#define NAME value`."""
    found = _find(r"^[ \t]*#[ \t]*define[ \t]+\w+\(")
    assert not found, found


def test_dtype_dispatch_only_in_common():
    found = [h for h in _find(r"switch \(dtype\)|case DVA_F32") if not h.startswith(COMMON)]
    assert not found, found


def test_workspace_rounding_only_in_common():
    found = [h for h in _find(r"\+ 255\) & ~") if not h.startswith(COMMON)]
    assert not found, found


# ---- unknown dtype / reduce codes: DVA_EINVAL, named after the entry point, nothing launched in their place
BAD_DTYPE, BAD_REDUCE = 7, 9
# the name an entry point's messages go by, where it is not the symbol without its dva_ prefix
LABEL = {"dva_segment_softmax_csr_fwd": "segment_softmax_fwd", "dva_segment_softmax_csr_bwd": "segment_softmax_bwd",
         "dva_heuristic_pool_fwd": "heuristic_pool"}
F32 = _lib.DVA_F32
SUM = 0


def _bufs():
    """Correctly sized fp32 buffers for every call below: a missing check launches a valid kernel on valid
    memory and fails the assertion, instead of reading bad addresses."""
    d = "cuda"
    f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=d)  # noqa: E731
    i = lambda *s: torch.zeros(*s, dtype=torch.int64, device=d)    # noqa: E731
    b = {"rows": f(8, 8), "seg": f(4, 8), "out_rows": f(8, 8), "out_seg": f(4, 8), "arg_seg": i(4, 8),
         "ptr": torch.arange(0, 10, 2, dtype=torch.int64, device=d), "idx": torch.arange(8, device=d),
         "arg4": i(4), "map3": f(8, 3), "ws": torch.zeros(1 << 20, dtype=torch.uint8, device=d),
         "fmap": f(1, 4, 4, 8), "gfmap": f(1, 4, 4, 8), "img": i(4),
         "pix": (torch.arange(16, dtype=torch.int32, device=d) % 4).reshape(8, 2),
         "vec": f(8), "vec2": f(8), "mean": f(8), "invstd": torch.ones(8, device=d), "dgb": f(2, 8),
         "labels": i(8), "lse": f(8), "loss": f(1), "stats": torch.ones(3, dtype=torch.int64, device=d),
         "compat": f(8, 4), "gcompat": f(8, 4), "smax": f(4, 4), "sden": torch.ones(4, 4, device=d),
         "sarg": torch.zeros(4, 4, dtype=torch.int32, device=d)}
    return b


def _calls(b, dtype, reduce):
    """(entry point, arguments without the stream); 4 segments / points of 2 rows each, 8 channels."""
    ws, nws = b["ws"], b["ws"].numel()
    pool = (b["img"], b["pix"], 0, b["ptr"])
    calls = [
        ("dva_segment_csr_fwd", b["rows"], b["ptr"], b["out_seg"], b["arg_seg"], 4, 8, 8, reduce, dtype),
        ("dva_segment_csr_bwd", b["seg"], b["ptr"], b["arg_seg"], b["out_rows"], 4, 8, 8, reduce, dtype),
        ("dva_gather_pool_fwd", b["fmap"], 1, *pool, b["out_seg"], b["arg_seg"], 1, 8, 4, 4, 4, 8, reduce, dtype),
        ("dva_gather_pool_bwd", b["seg"], 1, *pool, b["arg_seg"], b["gfmap"], 1, 8, 4, 4, 4, 8, reduce, dtype),
        ("dva_interp_pool_fwd", b["fmap"], 1, *pool, b["out_seg"], b["arg_seg"], 1, 8, 4, 4, 8, 8, 4, 8, reduce,
         dtype),
        ("dva_interp_pool_bwd", b["seg"], 1, *pool, b["arg_seg"], b["gfmap"], 1, 8, 4, 4, 8, 8, 4, 8, reduce, dtype),
        ("dva_gather_pool_bwd_det", b["seg"], 1, *pool, b["arg_seg"], b["gfmap"], 1, 8, 4, 4, 4, 8, reduce, dtype,
         ws, nws),
        ("dva_interp_pool_bwd_det", b["seg"], 1, *pool, b["arg_seg"], b["gfmap"], 1, 8, 4, 4, 8, 8, 4, 8, reduce,
         dtype, ws, nws),
    ]
    if reduce != SUM:
        return calls
    return calls + [
        ("dva_gather_csr", b["seg"], b["ptr"], b["out_rows"], 4, 8, 8, dtype),
        ("dva_segment_softmax_csr_fwd", b["rows"], b["ptr"], b["out_rows"], 4, 8, 8, 1e-12, 1, dtype),
        ("dva_segment_softmax_csr_bwd", b["rows"], b["rows"], b["ptr"], b["out_rows"], 4, 8, 8, 1, dtype),
        ("dva_heuristic_pool_fwd", b["rows"], b["map3"], 3, 0, b["ptr"], b["out_seg"], b["arg4"], 4, 8, 8, 1, dtype),
        ("dva_scatter_add_rows", b["rows"], b["idx"], b["out_rows"], 8, 8, 8, dtype),
        ("dva_scatter_add_rows_det", b["rows"], b["idx"], b["out_rows"], 8, 8, 8, dtype, ws, nws),
        ("dva_transpose_last2", b["rows"], b["out_rows"], 1, 8, 8, dtype),
        ("dva_bn_act_fwd", b["rows"], None, None, b["vec"], b["vec2"], b["mean"], b["invstd"], b["out_rows"], 8, 8,
         1e-5, 0.1, 0.2, 1, dtype, ws, nws),
        ("dva_bn_act_bwd", b["rows"], b["rows"], None, None, b["mean"], b["invstd"], b["out_rows"], b["dgb"], 8, 8,
         0.2, 1, dtype, ws, nws),
        ("dva_csr_nll_fwd", b["rows"], dtype, b["labels"], None, 8, 8, 8, -1, b["lse"], b["loss"], b["stats"], ws,
         nws),
        ("dva_csr_nll_bwd", b["rows"], dtype, b["labels"], None, 8, 8, 8, -1, b["lse"], b["loss"], b["stats"],
         b["out_rows"]),
        ("dva_view_attention_fwd", b["rows"], None, 0, b["compat"], b["ptr"], None, None, b["out_seg"], None, None,
         None, None, 4, 8, 8, 8, 4, 1, 1e-12, dtype),
        ("dva_view_attention_bwd", b["rows"], None, 0, b["compat"], b["ptr"], None, None, b["seg"], b["smax"],
         b["sden"], b["sarg"], b["out_rows"], b["gcompat"], None, 0, 4, 8, 8, 8, 4, 1, dtype, None, 0),
    ]


@pytest.mark.gpu
@pytest.mark.parametrize("code", ["dtype", "reduce"])
def test_unknown_code_rejected(code):
    b = _bufs()
    calls = _calls(b, BAD_DTYPE, SUM) if code == "dtype" else _calls(b, F32, BAD_REDUCE)
    lib = _lib.load()
    bad = []
    for name, *args in calls:
        n0 = _lib.launch_count()
        rc = getattr(lib, name)(*[_lib.ptr(a) if isinstance(a, torch.Tensor) else a for a in args], _lib.stream_ptr())
        msg = _lib.last_error()
        label = LABEL.get(name, name[len("dva_"):])
        if rc != _lib.DVA_EINVAL or not msg.startswith(label + ":") or f"unknown {code}" not in msg:
            bad.append((name, rc, msg))
        elif name != "dva_heuristic_pool_fwd" and _lib.launch_count() != n0:
            bad.append((name, "launched", _lib.launch_count() - n0))
    torch.cuda.synchronize()
    assert not bad, bad
