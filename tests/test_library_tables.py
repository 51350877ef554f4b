"""Checks, without a GPU, over the records of _lib.LIBRARIES (file, signatures, header, kernel namespace, linked or
not) and the kernel tables of the linked libraries (tests/test_{eval,conv2d,unet,resnet18}_matrix_table.py):
  * each table holds exactly the kernels compiled into its library, all of them in the record's namespace;
  * no kernel family of a linked library appears in any other library;
  * each header under include/, its signatures dict and the library's exports agree, no entry point is declared by
    two libraries, and _lib.entry finds every entry point in the library that declares it;
  * each library is loaded once per process, and a linked library refuses to load beside a DVA_B200_LIB variant."""
import itertools
import os
import re
import subprocess
import sys

import pytest

from conftest import ROOT
from deepviewagg_b200 import _lib
import test_conv2d_matrix_table
import test_eval_matrix_table
import test_resnet18_matrix_table
import test_unet_matrix_table
from test_loss_matrix_table import demangled_kernels

# linked library -> (its kernel table's module, the number of kernels it compiles)
TABLES = {_lib.EVAL: (test_eval_matrix_table, 9), _lib.CONV: (test_conv2d_matrix_table, 18),
          _lib.UNET: (test_unet_matrix_table, 12), _lib.RESNET: (test_resnet18_matrix_table, 14)}
LINKED = [rec for rec in _lib.LIBRARIES if rec.linked]
LOADERS = {_lib.B200: "load", _lib.EVAL: "load_eval", _lib.CONV: "load_conv", _lib.UNET: "load_unet",
           _lib.RESNET: "load_resnet"}


def _short(rec):
    return rec.file.removeprefix("libdva_").removesuffix(".so")      # libdva_conv2d.so -> conv2d


linked = pytest.mark.parametrize("rec", LINKED, ids=_short)


def _built(rec):
    for p in (_lib.LIB_PATH, rec.path):
        if not os.path.exists(p):
            pytest.fail(f"{p} is not built")
    return rec.path


def test_records_cover_every_library():
    assert set(TABLES) == set(LINKED) and set(LOADERS) == set(_lib.LIBRARIES)
    assert [rec.file for rec in _lib.LIBRARIES if not rec.linked] == ["libdva_b200.so"]


@linked
def test_table_matches_library(rec):
    table, count = TABLES[rec]
    assert table.NAMESPACE == rec.namespace
    names = [n for n in demangled_kernels(_built(rec)) if "__internal" not in n]    # libdevice's static slow paths
    outside = sorted(n for n in names if not n.replace("void ", "", 1).startswith(rec.namespace))
    assert not outside, outside
    built = {table.canonical(n) for n in names}
    assert None not in built, names
    assert built == set(table.TABLE), {"compiled without a case": sorted(built - set(table.TABLE)),
                                       "case without a kernel": sorted(set(table.TABLE) - built)}
    assert len(table.TABLE) == count


@linked
def test_no_kernel_family_shared_with_the_other_libraries(rec):
    table, _ = TABLES[rec]
    ours = {table.canonical(n).split("<")[0] for n in demangled_kernels(_built(rec)) if table.canonical(n)}
    assert ours == set(table.FAMILIES)
    for other in _lib.LIBRARIES:
        if other is rec:
            continue
        names = {n.replace("void ", "", 1).split("(")[0] for n in demangled_kernels(_built(other))}
        assert not any(n.startswith(rec.namespace) for n in names), other.file
        assert not {n for n in names if n.split("::")[-1].split("<")[0] in ours}, other.file


def _declared(header):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(re.findall(r"\b(dva_[a-z0-9_]+)\s*\(", text))


@pytest.mark.parametrize("rec", _lib.LIBRARIES, ids=_short)
def test_header_signatures_and_exports_agree(rec):
    _built(rec)
    names = _declared(rec.header)
    assert names == set(rec.signatures)
    assert all(n.startswith(rec.namespace.replace("::", "_")) for n in names)
    lib = _lib.load_library(rec)
    for n in names:
        assert hasattr(lib, n), n
        assert _lib.entry(n) is getattr(lib, n)


def test_no_entry_point_in_two_libraries():
    for a, b in itertools.combinations(_lib.LIBRARIES, 2):
        assert not set(a.signatures) & set(b.signatures), (a.file, b.file)


@linked
def test_canonical_names_of_every_family(rec):
    table, _ = TABLES[rec]
    for f in table.FAMILIES:
        assert table.canonical(f"void {rec.namespace}{f}<float, 4>(float const*, long)") == f"{f}<float, 4>"
        assert table.canonical(f" {rec.namespace}{f}(float const*) ") == f
        for other in _lib.LIBRARIES:
            if other is not rec:
                assert table.canonical(f"void {other.namespace}{f}(float const*)") is None
    assert table.canonical(f"void {rec.namespace}not_a_family_kernel(float const*)") is None


def test_each_library_is_loaded_once():
    for rec, loader in LOADERS.items():
        lib = getattr(_lib, loader)()
        assert getattr(_lib, loader)() is lib and _lib.load_library(rec) is lib


def test_linked_libraries_refuse_a_variant_base_library(tmp_path):
    """In a fresh process, so that this one's loaded libraries stay as they are."""
    variant = str(tmp_path / "libdva_b200.so")
    code = ("from deepviewagg_b200 import _lib\n"
            f"for loader in {[LOADERS[rec] for rec in LINKED]!r}:\n"
            "    try:\n"
            "        getattr(_lib, loader)()\n"
            "    except RuntimeError as e:\n"
            "        print(e)\n")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=dict(os.environ, DVA_B200_LIB=variant),
                         capture_output=True, text=True, check=True).stdout
    in_tree = os.path.join(ROOT, "deepviewagg_b200", "libdva_b200.so")
    assert out.splitlines() == [f"{rec.file} links against {in_tree}; it cannot run beside the variant "
                                f"DVA_B200_LIB={variant}" for rec in LINKED]
