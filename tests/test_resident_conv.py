"""Caller level: Runtime.np_convolve of secure integer, fixed-point and prime-field arrays, Runtime.np_roll by a secret
shift and a secure polynomial product and divmod (mpyc.secpols) under install(resident=True) print what the plain
reference prints (1 party and -M3).  Around the np_convolve and np_roll calls no array is turned into Python ints, and
the packs are pinned below."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import HERE, run, mode   # noqa: F401  (mode: fixture)

CONV = os.path.join(HERE, 'programs', 'resident_conv.py')
# packed arrays around the np_convolve calls: the public int array and the scaled public float array (2), plus, with 1
# party only, one inside each of the two np_trunc calls that follow the fixed-point products (runtime.py:2633); neither
# comes from a convolution
CONV_PACKED = {1: 4, 3: 2}
ROLL_PACKED = 1                  # np_fromlist(unit_vector(shift, N + 1)) (runtime.py:3306)


@pytest.fixture(autouse=True)
def k10_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k10.py: in 'oracle' mode the CPU stand-in backend then answers K7's
    to K10's calls too, so that convolutions take the same path as on a GPU (in 'cuda' mode it is run_installed.py
    unchanged)."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k10.py'))


def split(out):
    lines = out.splitlines()
    counts = {line.split(' ')[1]: json.loads(line.split(' ', 2)[2]) for line in lines if line.startswith('counts ')}
    return [line for line in lines if not line.startswith('counts ')], counts


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_conv_equals_the_reference_with_pinned_counts(mode, parties):
    want, _ = split(run(mode, CONV, (), ('off',), parties=parties))
    got, counts = split(run(mode, CONV, (), ('install', 'resident'), parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == 14 and got == want
    conv, roll = counts['conv'], counts['roll']
    assert conv['materialised'] == 0 and conv['packed'] == CONV_PACKED[parties]
    assert conv['limb_ops'] >= 10                      # ten convolutions, each on the limbs
    assert roll['materialised'] == 0 and roll['packed'] == ROLL_PACKED
    assert roll['limb_ops'] >= 1
