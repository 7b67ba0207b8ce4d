"""Caller level: 2 ** x and mpc.np_pow(3, x) of SecInt(32) arrays, mpc.np_exp2 and mpc.np_exp of SecFxp(32) arrays and
np_pow(2, x) over GF(2^128 - 173) under install(resident=True) print what the plain reference prints (1 party and -M3; with
several parties the integral exponents are SecFxp, see tests/programs/resident_powexp.py).  Every gmpy.powmod_exp_list call
of Runtime._np_pow_public_int_base_secret_integral_exponent goes to K12, and the conversions around each call are pinned:
the opened c = b + r is settled once (the protocol reads `c.value >> f` and maps int over powmod_exp_list's result, which
no hook reaches) and, for the plain powers, the result is packed once."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import HERE, run, mode   # noqa: F401  (mode: fixture)

POWEXP = os.path.join(HERE, 'programs', 'resident_powexp.py')
CALLS = ('pow2', 'np_pow3', 'exp2', 'exp', 'pow2_p128')


@pytest.fixture(autouse=True)
def k12_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k12.py: in 'oracle' mode the CPU stand-in backend then answers K7's
    to K12's calls too (in 'cuda' mode it is run_installed.py unchanged)."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k12.py'))


def split(out):
    lines = out.splitlines()
    counts = {line.split(' ')[1]: json.loads(line.split(' ', 2)[2]) for line in lines if line.startswith('counts ')}
    lists = {line.split(' ')[1]: int(line.split(' ')[2]) for line in lines if line.startswith('lists ')}
    return [line for line in lines if not line.startswith('counts ')], counts, lists


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_powexp_equals_the_reference_with_pinned_counts(mode, parties):
    want, _, _ = split(run(mode, POWEXP, (), ('off',), parties=parties))
    got, counts, lists = split(run(mode, POWEXP, (), ('install', 'resident'), parties=parties,
                                   env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == 2 * len(CALLS) and got == want
    for name in CALLS:
        # party 0 draws r (one call) or not, as the protocol's sender rotation has it, and exponentiates the opened c
        assert lists[name] in (1, 2) and (parties == 3 or lists[name] == 2), name
        assert counts[name]['pow_exp'] == lists[name], name
        assert counts[name]['materialised'] == 1, name
        if name not in ('exp2', 'exp'):
            assert counts[name]['packed'] == 1, name
