"""Caller level: secure-array sums (np_sum, np_cumsum, np_cumulative_sum, np_outer) under install(resident=True) print
what the plain reference prints, with no Python ints made between input and output; and the demos that sum and take
outer products of secure arrays (np_id3gini, np_lpsolver) print the same results installed as uninstalled."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import DEMOS_DIR, HERE, run, mode, trim_for_gpu   # noqa: F401  (mode: fixture)

PROGRAM = os.path.join(HERE, 'programs', 'resident_sums.py')


@pytest.fixture(autouse=True)
def k7_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k7.py: in 'oracle' mode the CPU stand-in backend then answers K7's
    calls too, so that the sums take the same path as on a GPU (in 'cuda' mode it is run_installed.py unchanged)."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k7.py'))


def split(out):
    lines = out.splitlines()
    between = [json.loads(line.split(' ', 1)[1]) for line in lines if line.startswith('between ')]
    return [line for line in lines if not line.startswith('between ')], between


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_sums_equal_the_reference(mode, parties):
    want, _ = split(run(mode, PROGRAM, (), ('off',), parties=parties))
    got, between = split(run(mode, PROGRAM, (), ('install', 'resident'), parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == 12 and got == want
    assert between and between[0]['materialised'] == 0 and between[0]['packed'] == 0
    assert between[0]['limb_ops'] >= 12


@pytest.mark.parametrize('demo, args', [('np_id3gini.py', ['-i', '1']), ('np_lpsolver.py', [])], ids=['np_id3gini', 'np_lpsolver'])
@pytest.mark.parametrize('parties', [1, 3])
def test_summing_demos_installed_equal_uninstalled(mode, demo, args, parties):
    if DEMOS_DIR is None or not os.path.isfile(os.path.join(DEMOS_DIR, demo)):
        pytest.skip('reference demos/ not available (package-only reference)')
    trim_for_gpu(mode, parties == 3)
    want = run(mode, demo, args, ('off',), cwd=DEMOS_DIR, parties=parties)
    got = run(mode, demo, args, ('install', 'resident'), cwd=DEMOS_DIR, parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'})
    strip = lambda s: [line for line in s.splitlines() if 'elapsed time' not in line.lower() and 'bytes' not in line.lower()]   # noqa: E731
    assert strip(got) == strip(want)
