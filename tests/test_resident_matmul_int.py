"""Caller level: mpc.np_matmul with public int64 operands on either side, np_argmax / np_argmin, np_unit_vector, a SecFxp
product with a public float matrix and np.matmul of opened field arrays, under install(resident=True, public_matmul=True),
print what the plain reference prints (1 party and -M3).  None of these calls settles an operand at a matmul: the
integer-operand products run on K14, np.matmul of field arrays on K1c.  Each window also holds the output() that opens its result, hence the settles
counted in 'materialised' (the opened values, and in argmax / argmin / unit_vector the comparison protocols' own openings);
the one-element result of np_unit_vector's 1-D @ 1-D product is the only settle inside resident.matmul.  The float matrix
reaches matmul as an object array of ints (np_matmul rounds it), so that product stays on K1c."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import HERE, run, mode   # noqa: F401  (mode: fixture)

PROGRAM = os.path.join(HERE, 'programs', 'resident_matmul_int.py')
CALLS = ('matmul_xW', 'matmul_Wx', 'matmul_xv', 'argmax', 'argmin', 'unit_vector', 'fxp_float_left', 'np_matmul_opened')


@pytest.fixture(autouse=True)
def k14_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k14.py: install(public_matmul=True), and in 'oracle' mode the CPU
    stand-in backend answers K7's to K14's calls too."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k14.py'))


def split(out):
    lines = out.splitlines()
    counts = {line.split(' ')[1]: json.loads(line.split(' ', 2)[2]) for line in lines if line.startswith('counts ')}
    return [line for line in lines if not line.startswith('counts ')], counts


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_matmul_int_equals_the_reference_with_pinned_counts(mode, parties):
    want, _ = split(run(mode, PROGRAM, (), ('off',), parties=parties))
    got, counts = split(run(mode, PROGRAM, (), ('install', 'resident'), parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == len(CALLS) and got == want
    for name in CALLS:
        assert counts[name]['matmul_settles'] == 0, name
        assert counts[name]['inner_settles'] == (name == 'unit_vector'), name
    for name in CALLS[:6]:
        assert counts[name]['matmul_int'] == 1, name
    for name in CALLS[6:]:
        assert counts[name]['matmul_int'] == 0 and counts[name]['limb_ops'] >= 1, name
    assert counts['np_matmul_opened']['materialised'] == 0
    for name in CALLS[:3]:
        assert counts[name]['materialised'] == 1, name                 # output() of the result
