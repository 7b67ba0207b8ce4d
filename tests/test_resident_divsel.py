"""Caller level: == and != of SecInt(64) arrays (Runtime._np_is_zero), Runtime.np_reciprocal, / of SecInt(32) and
SecFld(2^61 - 1) arrays, np_divide by a public field array, np_lsb and np_from_bits under install(resident=True) print what
the plain reference prints (1 party and -M3).  No call turns an array into Python ints, and the packs are pinned below."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import HERE, run, mode   # noqa: F401  (mode: fixture)

DIVSEL = os.path.join(HERE, 'programs', 'resident_divsel.py')
CALLS = ('eq', 'ne', 'reciprocal', 'int_div', 'fld_div', 'public_div', 'lsb', 'from_bits')
# packs per call; none is of a value that was ever limb-backed:
#   eq, lsb  with 1 party, np_random_bits' public row of random bits (runtime.py:4251, `field.array(_r.value**2 + z.value)`
#            gets the public ints of the one-party PRSS zero sharing)
#   ne       as eq, plus np_subtract's public 1 in `1 - (x == y)` (runtime.py:1058)
#   public_div  np_divide's `field.array(b)` of the public divisor (runtime.py:1218)
PACKED = {1: {'eq': 1, 'ne': 2, 'lsb': 1, 'public_div': 1}, 3: {'ne': 1, 'public_div': 1}}


@pytest.fixture(autouse=True)
def k11_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k11.py: in 'oracle' mode the CPU stand-in backend then answers K7's
    to K11's calls too, so that division and selection take the same path as on a GPU (in 'cuda' mode it is
    run_installed.py unchanged)."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k11.py'))


def split(out):
    lines = out.splitlines()
    counts = {line.split(' ')[1]: json.loads(line.split(' ', 2)[2]) for line in lines if line.startswith('counts ')}
    return [line for line in lines if not line.startswith('counts ')], counts


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_divsel_equals_the_reference_with_pinned_counts(mode, parties):
    want, _ = split(run(mode, DIVSEL, (), ('off',), parties=parties))
    got, counts = split(run(mode, DIVSEL, (), ('install', 'resident'), parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == len(CALLS) and got == want
    for name in CALLS:
        assert counts[name]['materialised'] == 0, name
        assert counts[name]['packed'] == PACKED[parties].get(name, 0), name
        assert counts[name]['limb_ops'] >= 1, name
    assert counts['eq']['limb_ops'] >= 3 and counts['ne']['limb_ops'] >= 3     # two np.where selections and is_sqr
