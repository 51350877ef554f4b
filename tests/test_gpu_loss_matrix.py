"""Every kernel of tests/test_loss_matrix_table.py launched and proven launched: each scenario runs once under the
kernel recorder of tests/test_gpu_kernel_matrix.py and checks its results against the references and bounds of the
table's module docstring; each case asserts, by name, that its kernel ran in its scenario."""
import functools

import pytest

from test_gpu_kernel_matrix import record
from test_gpu_sparseconv3d import lovasz_scenario, wnll_scenario
from test_kernel_matrix_table import DTYPES
from test_loss_matrix_table import CASE_IDS, CASES, TABLE, canonical

pytestmark = pytest.mark.gpu
SEEN = set()
WANT = {}
for _c in CASES:
    WANT.setdefault(_c["scenario"], set()).add(_c["kernel"])

SCENARIO_FNS = {}
for _dt in DTYPES:
    SCENARIO_FNS[f"wnll_{_dt}"] = functools.partial(wnll_scenario, _dt)
    SCENARIO_FNS[f"lovasz_{_dt}"] = functools.partial(lovasz_scenario, _dt)

_RESULTS = {}


def run_scenario(name):
    """Run a scenario once per session under the recorder; its checks raise on a wrong result."""
    if name not in _RESULTS:
        try:
            _, names = record(SCENARIO_FNS[name], tuple(WANT[name]), canon=canonical, seen=SEEN)
            _RESULTS[name] = (names, None)
        except AssertionError as e:
            _RESULTS[name] = (set(), e)
    names, err = _RESULTS[name]
    if err is not None:
        raise err
    return names


def test_every_scenario_has_a_function():
    assert set(WANT) <= set(SCENARIO_FNS), sorted(set(WANT) - set(SCENARIO_FNS))


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_kernel(case):
    names = run_scenario(case["scenario"])
    assert case["kernel"] in names, f"{case['kernel']} did not run in {case['scenario']}; recorded: {sorted(names)}"


def test_every_kernel_launched():
    """The union of the kernels recorded by all scenarios is exactly the table."""
    for name in WANT:
        try:
            run_scenario(name)
        except AssertionError:
            pass
    table = set(TABLE)
    assert SEEN == table, {"never launched": sorted(table - SEEN), "launched without a case": sorted(SEEN - table)}
