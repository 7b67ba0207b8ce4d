"""The fields of MPyC's default secure types (tests/mpyc_fields.py): each literal is the reference's find_prime_root for
its bit length, and ff_arith.cuh's reduction family for it -- compiled on the host by tests/native/host_check.cpp -- picks
the expected (kind, limbs, bits) and agrees with Python integers on products, sums, lazy sums at their bound, small-factor
reductions and powers.  Only the moduli that tests/arith_vectors.py does not already cover are run through the checker."""
import os
import shutil
import subprocess
import sys

import pytest

from arith_vectors import PRIMES as ARITH_PRIMES, commands, expected_kind
from mpyc_fields import FIELDS, field_id
from oracle import reference

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'native', 'host_check.cpp')
BIN = os.path.join(HERE, 'native', '_build', 'host_check_mpyc')


@pytest.fixture(scope='module')
def checker():
    if shutil.which('g++') is None:
        pytest.skip('g++ not available')
    os.makedirs(os.path.dirname(BIN), exist_ok=True)
    subprocess.run(['g++', '-std=c++17', '-O2', '-fno-strict-aliasing', '-x', 'c++', SRC, '-o', BIN], check=True)

    def run(lines):
        r = subprocess.run([BIN], input='\n'.join(lines) + '\n', capture_output=True, text=True, check=True)
        return r.stdout.split()
    return run


@pytest.fixture(scope='module')
def finfields():
    ref = reference.path()
    if ref is None:
        pytest.skip('reference not present ($MPYC_REFERENCE, or the copy build() makes in oracle/_ref)')
    sys.dont_write_bytecode = True
    sys.path.insert(0, ref)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    try:
        from mpyc import finfields
    finally:
        sys.argv = argv
    yield finfields
    sys.path.remove(ref)


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_literal_is_the_reference_prime(finfields, f):
    p, n, w = finfields.find_prime_root(f.bits, n=f.n)
    assert p == f.p and (p - 1) % n == 0 and n >= f.n
    assert pow(w, n, p) == 1


@pytest.mark.parametrize('f', FIELDS, ids=field_id)
def test_declared_kind_and_limbs(f):
    assert f.p.bit_length() == f.bits
    assert (expected_kind(f.p), (f.bits + 63) // 64) == (f.kind, f.limbs)


@pytest.mark.parametrize('f', [f for f in FIELDS if f.p not in ARITH_PRIMES], ids=field_id)
def test_field_arithmetic_on_host(checker, f):
    p = f.p
    lines, want, (L, k) = commands(p)
    out = checker(lines)
    kind, Lr, kr = (int(x) for x in out[:3])
    assert (kind, Lr, kr) == (f.kind, L, k) == (expected_kind(p), f.limbs, f.bits)
    got = out[3:]
    assert len(got) == len(want)
    bad = [(lines[i + 1], got[i], f'{want[i]:x}') for i in range(len(want)) if got[i] != f'{want[i]:x}']
    assert not bad, bad[:5]

