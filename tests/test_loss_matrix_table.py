"""Kernel matrix of the loss kernels of the sparse-conv models, namespace dva_loss:: -- the class-weighted CSR
log-softmax NLL (csr_nll.cu, csr_nll_w*) and the Lovász-softmax (lovasz.cu).

tests/test_gpu_loss_matrix.py runs every scenario on the GPU under the kernel recorder and asserts, by name, the
kernels each case must launch.  This file checks, without a GPU, that
  * the case table holds exactly the dva_loss:: kernels compiled into libdva_b200.so;
  * every kernel of the library, in any namespace, sits in exactly one of the four tables (the three dva:: tables
    of tests/test_kernel_matrix_table.py, tests/test_pool_gemm_matrix_table.py, tests/test_rest_matrix_table.py,
    and this one): a kernel anywhere that no table lists fails here.

References and bounds (u32 = 2^-24, u_s = half an ulp of the storage type, ke = 8 u32; tests/test_gpu_sparseconv3d.py):
  weighted NLL   float64 nll_loss(weight=w): the NLL row of tests/test_rest_matrix_table.py with the mean of mag_v
        weighted by w[y_v] and count replaced by W / w[y_v]:
        loss   |got - ref| <= ke (K + 2) sum_v w_v mag_v / W + u32 |ref|
        grad   u_s |ref| + ke ((K + 2) mag_v p_vj + 1) |g| w_v / W + tiny
  Lovász   oracle/lovasz_oracle.py (float64): loss within 2 u32 |ref|; on tie-free inputs the gradient within
        4 u32 |ref| + 1e-15; on tied inputs the sum over each tied block of grad * d|fg - p|/dp within
        u_s sum|ref| + n tiny + 4 u32 |ref sum|.
"""
import os
import shutil
import subprocess

import pytest

from test_kernel_matrix_table import CPP, DTYPES, _lib_path, kname, parse_kernel
import test_kernel_matrix_table as KM
import test_pool_gemm_matrix_table as PG
import test_rest_matrix_table as RM

NAMESPACE = "dva_loss::"
FAMILIES = ("csr_nll_wfwd_kernel", "csr_nll_wbwd_kernel", "csr_nll_wfinalize_kernel", "lovasz_keys_kernel",
            "lovasz_fg_kernel", "lovasz_loss_kernel", "lovasz_finalize_kernel", "lovasz_bwd_kernel")


def canonical(name):
    """Demangled dva_loss:: kernel name -> 'family<args>' (the form of the other tables); None otherwise."""
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

    def add(kernel, *scenarios):
        assert kernel not in c, kernel
        c[kernel] = list(scenarios)

    for dt in DTYPES:
        add(kname("csr_nll_wfwd_kernel", CPP[dt]), f"wnll_{dt}")
        add(kname("csr_nll_wbwd_kernel", CPP[dt]), f"wnll_{dt}")
        for log_probs in (False, True):
            add(kname("lovasz_keys_kernel", CPP[dt], log_probs), f"lovasz_{dt}")
            add(kname("lovasz_bwd_kernel", CPP[dt], log_probs), f"lovasz_{dt}")
    add("csr_nll_wfinalize_kernel", "wnll_f32")
    for k in ("lovasz_fg_kernel", "lovasz_loss_kernel", "lovasz_finalize_kernel"):
        add(k, "lovasz_f32")
    return c


TABLE = _cases()
CASES = [dict(kernel=k, scenario=s) for k, ss in TABLE.items() for s in ss]
CASE_IDS = [f"{c['kernel']}@{c['scenario']}" for c in CASES]


def demangled_kernels(lib_path):
    """Every demangled kernel symbol of the library (cuobjdump -symbols | c++filt)."""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "-symbols", lib_path], capture_output=True, text=True, check=True).stdout
    mangled = [ln.split()[-1] for ln in out.splitlines() if "STT_FUNC" in ln]
    dem = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout
    return [n for n in dem.splitlines() if n.strip()]


def _built():
    path = _lib_path()
    if not os.path.exists(path):
        pytest.fail(f"{path} is not built")
    return path


def test_case_table_matches_library():
    built = {k for k in (canonical(n) for n in demangled_kernels(_built())) if k is not None}
    table = set(TABLE)
    assert built == table, {"compiled without a case": sorted(built - table),
                            "case without a kernel": sorted(table - built)}
    assert len(table) == 22
    assert len(CASE_IDS) == len(set(CASE_IDS))


def test_four_tables_close_over_the_library():
    """Every kernel of the library, in any namespace, is in exactly one of the four tables: a dva_loss:: kernel in
    this one, a dva:: kernel in one of the other three (checked there), and no kernel outside both namespaces."""
    names = demangled_kernels(_built())
    outside = sorted(n for n in names
                     if not n.replace("void ", "", 1).startswith(("dva::", NAMESPACE))
                     and "__internal" not in n)            # libdevice's static slow paths, not kernels of ours
    assert not outside, outside
    loss = {k for k in (canonical(n) for n in names) if k is not None}
    unlisted = sorted(n for n in names if n.replace("void ", "", 1).startswith(NAMESPACE) and canonical(n) is None)
    assert not unlisted, unlisted
    dva_tables = set(KM.CASE_IDS) | set(PG.CASE_IDS) | set(RM.TABLE)
    assert not (loss & dva_tables)
    assert loss == set(TABLE)


def test_canonical_names():
    assert canonical("void dva_loss::lovasz_keys_kernel<__half, true>(__half const*, long const*, long, int, long, "
                     "float*)") == "lovasz_keys_kernel<__half, true>"
    assert canonical("dva_loss::lovasz_fg_kernel(float const*, long const*, long const*, long, int, unsigned char*, "
                     "int*)") == "lovasz_fg_kernel"
    assert canonical("void dva::csr_nll_fwd_kernel<float>(float const*)") is None
