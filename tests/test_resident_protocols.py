"""Caller level: the protocols that move arrays around between their GPU steps (np_sort, np_argmax, np_amax, np_add_bits,
max-pooling; tests/programs/resident_protocols.py) print what the plain reference prints under install(resident=True,
public_matmul=True), with the conversion counts pinned below (tests/test_resident_layout.py pins them without
public_matmul)."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import HERE, run, mode   # noqa: F401  (mode: fixture)

PROTOCOLS = os.path.join(HERE, 'programs', 'resident_protocols.py')
# (materialised, packed) between input and output of resident_protocols.py on party 0 with K8 and K14 (DESIGN.md section
# 5c names each one); without public_matmul the same runs have (2, 62) and (2, 47): K14 keeps np_argmax's
# `u @ np.arange(n)` operand limb-backed
PROTOCOL_COUNTS = {1: (1, 62), 3: (1, 47)}


@pytest.fixture(autouse=True)
def k14_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k14.py: install(public_matmul=True), and in 'oracle' mode the CPU
    stand-in backend answers K7's to K14's calls too, so that the protocols take the same path as on a GPU."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k14.py'))


def split(out):
    lines = out.splitlines()
    between = [json.loads(line.split(' ', 1)[1]) for line in lines if line.startswith('between ')]
    return [line for line in lines if not line.startswith('between ')], between


@pytest.mark.parametrize('parties', [1, 3])
def test_protocols_equal_the_reference_with_pinned_counts(mode, parties):
    want, _ = split(run(mode, PROTOCOLS, (), ('off',), parties=parties))
    got, between = split(run(mode, PROTOCOLS, (), ('install', 'resident'), parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == 5 and got == want
    assert (between[0]['materialised'], between[0]['packed']) == PROTOCOL_COUNTS[parties]
