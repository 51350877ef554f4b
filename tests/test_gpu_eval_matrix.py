"""Every kernel of tests/test_eval_matrix_table.py launched and proven launched: each scenario of
tests/test_gpu_metrics.py runs once under the kernel recorder of tests/test_gpu_kernel_matrix.py, checks its
results for equality, and each case asserts, by name, that its kernel ran."""
import functools

import pytest

from test_eval_matrix_table import TABLE, canonical
from test_gpu_kernel_matrix import record
from test_gpu_metrics import nn_scenario, pred_scenario, scores_scenario, vote_scenario
from test_kernel_matrix_table import DTYPES

pytestmark = pytest.mark.gpu
SEEN = set()
WANT = {}
for _k, _s in TABLE.items():
    WANT.setdefault(_s, set()).add(_k)

SCENARIO_FNS = {"pred": pred_scenario, "nn": functools.partial(nn_scenario, N=20_000)}
for _dt in DTYPES:
    SCENARIO_FNS[f"scores_{_dt}"] = functools.partial(scores_scenario, _dt, n=50_000)
    SCENARIO_FNS[f"vote_{_dt}"] = functools.partial(vote_scenario, _dt, N=50_000, n=10_000)

_RESULTS = {}


def run_scenario(name):
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


@pytest.mark.parametrize("kernel", sorted(TABLE))
def test_kernel(kernel):
    names = run_scenario(TABLE[kernel])
    assert kernel in names, f"{kernel} did not run in {TABLE[kernel]}; recorded: {sorted(names)}"


def test_every_kernel_launched():
    for name in WANT:
        try:
            run_scenario(name)
        except AssertionError:
            pass
    assert SEEN == set(TABLE), {"never launched": sorted(set(TABLE) - SEEN),
                                "launched without a case": sorted(SEEN - set(TABLE))}
