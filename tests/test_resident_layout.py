"""Caller level: views, writes, transposes, joins, flips, rolls and broadcasts of secure arrays under install(resident=True)
print what the plain reference prints, with no Python ints made between input and output; and the protocols that move
arrays around between their GPU steps (np_sort, np_argmax, np_amax, np_add_bits, max-pooling) print the same results
with the conversion counts pinned below."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import HERE, run, mode   # noqa: F401  (mode: fixture)

LAYOUT = os.path.join(HERE, 'programs', 'resident_layout.py')
PROTOCOLS = os.path.join(HERE, 'programs', 'resident_protocols.py')
# (materialised, packed) between input and output of resident_protocols.py on party 0 with K8 (DESIGN.md section 5c
# names each one); before K8 the same runs had (34, 156) and (35, 139)
PROTOCOL_COUNTS = {1: (2, 62), 3: (2, 47)}


@pytest.fixture(autouse=True)
def k8_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k8.py: in 'oracle' mode the CPU stand-in backend then answers K7's
    and K8's calls too, so that layout takes the same path as on a GPU (in 'cuda' mode it is run_installed.py unchanged)."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k8.py'))


def split(out):
    lines = out.splitlines()
    between = [json.loads(line.split(' ', 1)[1]) for line in lines if line.startswith('between ')]
    return [line for line in lines if not line.startswith('between ')], between


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_layout_equals_the_reference(mode, parties):
    want, _ = split(run(mode, LAYOUT, (), ('off',), parties=parties))
    got, between = split(run(mode, LAYOUT, (), ('install', 'resident'), parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == 17 and got == want
    assert between and between[0]['materialised'] == 0 and between[0]['packed'] == 0
    assert between[0]['limb_ops'] >= 17


@pytest.mark.parametrize('parties', [1, 3])
def test_protocols_equal_the_reference_with_pinned_counts(mode, parties):
    want, _ = split(run(mode, PROTOCOLS, (), ('off',), parties=parties))
    got, between = split(run(mode, PROTOCOLS, (), ('install', 'resident'), parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == 5 and got == want
    assert (between[0]['materialised'], between[0]['packed']) == PROTOCOL_COUNTS[parties]
