"""Caller level: Runtime.np_det of a secure integer matrix and np.linalg.det / solve / inv / matrix_power of opened
products under install(resident=True) print what the plain reference prints (1 party and -M3).  The public np.linalg calls
on the opened, limb-backed arrays make no Python ints (0 settles, 0 packs), and the counts of the whole np_det call are
pinned below; DESIGN.md section 5c names each one, and none of them is the opened L @ (U @ A)."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import HERE, run, mode   # noqa: F401  (mode: fixture)

LINALG = os.path.join(HERE, 'programs', 'resident_linalg.py')
# (materialised, packed) of one mpc.np_det call on party 0: np.diag of the random factor U settles it (finfields.py:982,
# runtime.py:3966), and the triangular factors L and U built from its ints are packed by L @ (U @ A) (:3978)
NP_DET_COUNTS = {1: (1, 2), 3: (1, 2)}


@pytest.fixture(autouse=True)
def k9_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k9.py: in 'oracle' mode the CPU stand-in backend then answers K7's,
    K8's and K9's calls too, so that linear algebra takes the same path as on a GPU (in 'cuda' mode it is run_installed.py
    unchanged)."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k9.py'))


def split(out):
    lines = out.splitlines()
    counts = {line.split(' ')[1]: json.loads(line.split(' ', 2)[2]) for line in lines if line.startswith('counts ')}
    return [line for line in lines if not line.startswith('counts ')], counts


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_linalg_equals_the_reference_with_pinned_counts(mode, parties):
    want, _ = split(run(mode, LINALG, (), ('off',), parties=parties))
    got, counts = split(run(mode, LINALG, (), ('install', 'resident'), parties=parties, env_extra={'MPYC_B200_OPS_MIN_SIZE': '1'}))
    assert len(want) == 9 and got == want
    public, det = counts['public'], counts['np_det']
    assert (public['materialised'], public['packed']) == (0, 0)
    assert public['limb_ops'] == 8                     # det, stacked det, solve, inv and four powers, all on the limbs
    assert (det['materialised'], det['packed']) == NP_DET_COUNTS[parties]
    assert det['limb_ops'] >= 3
