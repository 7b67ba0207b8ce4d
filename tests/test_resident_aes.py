"""Caller level for K15: tests/programs/resident_aes.py (a batched S-box and inverse S-box on 64 secret SecFld(2^8) bytes and one
AES-128 block) and demos/np_aes.py -M3 (AES-128 and AES-256, both directions) under install(resident=True) print what the
plain reference prints, with 1 party and -M3.  Between input and output the program settles nothing but the opened, public
`c` of each Runtime.np_to_bits call (`np.vectorize(int, otypes='O')(c.value)`, runtime.py:4421, which no hook reaches): one
per S-box, 20 in the AES block (10 rounds and 10 key-schedule words).  The pack and K15 call counts are pinned too; the packs
are the public affine matrix and vector, the integer bits `c_bits` of np_to_bits and the round constants."""
import json
import os

import pytest

import test_reference_runtime
from test_reference_runtime import DEMOS_DIR, HAVE_DEMOS, HERE, run, mode   # noqa: F401  (mode: fixture)

PROGRAM = os.path.join(HERE, 'programs', 'resident_aes.py')
EVERYTHING = {'MPYC_B200_OPS_MIN_SIZE': '1'}
FIPS197_128 = '69c4e0d86a7b0430d8cdb78070b4c55a'
FIPS197_256 = '8ea2b7ca516745bfeafc49904b496089'
# step -> (c_settles, packed, K15 calls), the same with 1 party and -M3
COUNTS = {'sbox': (1, 4, 6), 'inv_sbox': (1, 4, 6), 'aes128': (20, 108, 120)}


@pytest.fixture(autouse=True)
def k15_launcher(monkeypatch):
    """Every party starts through tests/run_installed_k15.py: in 'oracle' mode the CPU stand-in backend answers K7's to
    K15's calls too."""
    monkeypatch.setattr(test_reference_runtime, 'LAUNCHER', os.path.join(HERE, 'run_installed_k15.py'))


def split(out):
    lines = out.splitlines()
    counts = {line.split(' ')[1]: json.loads(line.split(' ', 2)[2]) for line in lines if line.startswith('counts ')}
    return [line for line in lines if not line.startswith('counts ')], counts


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_aes_equals_the_reference_with_pinned_counts(mode, parties):
    want, _ = split(run(mode, PROGRAM, ('64',), ('off',), parties=parties))
    got, counts = split(run(mode, PROGRAM, ('64',), ('install', 'resident'), parties=parties, env_extra=EVERYTHING))
    assert got == want and len(got) == 3
    assert got[0].startswith('sbox 637c777bf26b6fc5') and got[1].startswith('inv_sbox 52096ad53036a538')
    assert got[2] == f'aes128 {FIPS197_128}'
    for name, (c_settles, packed, k15) in COUNTS.items():
        cnt = counts[name]
        assert cnt['other_settles'] == 0, name
        assert cnt['c_settles'] == cnt['materialised'] == c_settles, name
        assert cnt['packed'] == packed, name
        assert cnt['gf_local'] == k15, name


def test_np_aes_demo_three_parties_equals_the_reference(mode):
    """demos/np_aes.py -M3 unchanged: the reference's ciphertexts and plaintexts, and the same lines under install(resident=True)."""
    if not HAVE_DEMOS:
        pytest.skip('reference demos/ not available (package-only reference)')
    want = run(mode, 'np_aes.py', (), ('off',), cwd=DEMOS_DIR, parties=3)
    got = run(mode, 'np_aes.py', (), ('install', 'resident'), cwd=DEMOS_DIR, parties=3, env_extra=EVERYTHING)
    assert f'Ciphertext:  {FIPS197_128}' in want and f'Ciphertext:  {FIPS197_256}' in want
    assert want.count('Plaintext:   00112233445566778899aabbccddeeff') == 3
    assert got == want
