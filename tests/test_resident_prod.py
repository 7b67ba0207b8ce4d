"""Caller level: mpc.np_is_zero_public and x < y of SecInt(16) arrays, and np.prod / FiniteFieldArray.prod / np.cumprod /
np.cumulative_prod / np.all / np.any of arrays opened with output(raw=True), under install(resident=True) print what the
plain reference prints (1 party and -M3).  SecInt(16) lives in a 48-bit field, below 2 * sec_param bits, so
Runtime.np_is_zero_public tests its opened r * s with `np.all(...)` (runtime.py:965): that test now runs on K13's count and
settles nothing, and neither does any other call below."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import HERE, run, mode   # noqa: F401  (mode: fixture)

PROD = os.path.join(HERE, 'programs', 'resident_prod.py')
CALLS = ('is_zero_public', 'lt', 'prod', 'prod_all', 'prod_method', 'cumprod', 'cumulative_prod', 'all', 'any', 'all_none',
         'any_none')


@pytest.fixture(autouse=True)
def k13_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k13.py: in 'oracle' mode the CPU stand-in backend then answers K7's
    to K13's calls too (in 'cuda' mode it is run_installed.py unchanged)."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k13.py'))


def split(out):
    lines = out.splitlines()
    counts = {line.split(' ')[1]: json.loads(line.split(' ', 2)[2]) for line in lines if line.startswith('counts ')}
    return [line for line in lines if not line.startswith('counts ')], counts


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_prod_equals_the_reference_with_pinned_counts(mode, parties):
    want, _ = split(run(mode, PROD, (), ('off',), parties=parties))
    got, counts = split(run(mode, PROD, (), ('install', 'resident'), parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == len(CALLS) and got == want
    for name in CALLS:
        assert counts[name]['materialised'] == 0, name
        assert counts[name]['zero_test_settles'] == 0, name
    for name in CALLS[2:]:
        assert counts[name]['prod'] == 1, name
    # np_is_zero_public's np.all and the np.all inside the comparison's zero test ran on K13
    assert counts['is_zero_public']['prod'] >= 1 and counts['lt']['prod'] >= 1
