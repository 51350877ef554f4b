"""Every kernel of the single-scenario kernel tables launched and proven launched: each library's scenario (checked
against float64 in its own test file) runs once under the kernel recorder of tests/test_gpu_kernel_matrix.py, and
each case asserts, by name, that its kernel ran."""
import pytest

import test_conv2d_matrix_table
import test_resnet18_matrix_table
import test_unet_matrix_table
from test_gpu_image_encoder import encoder_scenario
from test_gpu_image_resnet18 import resnet_scenario
from test_gpu_image_unet import unet_scenario
from test_gpu_kernel_matrix import record

pytestmark = pytest.mark.gpu
# library -> (its kernel table's module, the scenario that launches every kernel of the table)
LIBRARIES = {"conv2d": (test_conv2d_matrix_table, encoder_scenario),
             "unet": (test_unet_matrix_table, unet_scenario),
             "resnet18": (test_resnet18_matrix_table, resnet_scenario)}
SEEN = {lib: set() for lib in LIBRARIES}
_RESULT = {}


def names(lib):
    if lib not in _RESULT:
        table, scenario = LIBRARIES[lib]
        _, _RESULT[lib] = record(scenario, tuple(table.TABLE), canon=table.canonical, seen=SEEN[lib])
    return _RESULT[lib]


@pytest.mark.parametrize("lib,kernel", [(lib, k) for lib, (table, _) in LIBRARIES.items() for k in sorted(table.TABLE)])
def test_kernel(lib, kernel):
    assert kernel in names(lib), f"{kernel} did not run; recorded: {sorted(names(lib))}"


@pytest.mark.parametrize("lib", LIBRARIES)
def test_every_kernel_launched(lib):
    table, _ = LIBRARIES[lib]
    names(lib)
    assert SEEN[lib] == set(table.TABLE), {"never launched": sorted(set(table.TABLE) - SEEN[lib]),
                                           "launched without a case": sorted(SEEN[lib] - set(table.TABLE))}
