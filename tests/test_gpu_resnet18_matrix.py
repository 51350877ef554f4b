"""Every kernel of tests/test_resnet18_matrix_table.py launched and proven launched: the Pyramid scenario of
tests/test_gpu_image_resnet18.py runs once under the kernel recorder of tests/test_gpu_kernel_matrix.py, and each
case asserts, by name, that its kernel ran."""
import pytest

from test_gpu_image_resnet18 import resnet_scenario
from test_gpu_kernel_matrix import record
from test_resnet18_matrix_table import TABLE, canonical

pytestmark = pytest.mark.gpu
SEEN = set()
_RESULT = {}


def names():
    if "names" not in _RESULT:
        _, _RESULT["names"] = record(resnet_scenario, tuple(TABLE), canon=canonical, seen=SEEN)
    return _RESULT["names"]


@pytest.mark.parametrize("kernel", sorted(TABLE))
def test_kernel(kernel):
    assert kernel in names(), f"{kernel} did not run; recorded: {sorted(names())}"


def test_every_kernel_launched():
    names()
    assert SEEN == set(TABLE), {"never launched": sorted(set(TABLE) - SEEN),
                                "launched without a case": sorted(SEEN - set(TABLE))}
