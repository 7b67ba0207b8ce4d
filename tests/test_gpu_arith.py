"""Device-side check of the multi-limb primitives: tests/native/dev_check.cu runs the templates of
mpyc_b200/csrc/ff_arith.cuh inside a kernel (PTX carry chains, IMAD.WIDE pairs) on the same command
streams as the host checker; results must equal Python integer arithmetic."""
import os
import shutil
import subprocess

import pytest

from arith_vectors import PRIMES, commands, expected_kind

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'native', 'dev_check.cu')
BIN = os.path.join(HERE, 'native', '_build', 'dev_check')


@pytest.fixture(scope='module')
def checker():
    torch = pytest.importorskip('torch')
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    hdr = os.path.join(HERE, '..', 'mpyc_b200', 'csrc', 'ff_arith.cuh')
    if not os.path.exists(BIN) or os.path.getmtime(BIN) < max(os.path.getmtime(SRC), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(BIN), exist_ok=True)
        subprocess.run([nvcc, '-std=c++17', '-O3', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', BIN, SRC], check=True)

    def run(lines):
        r = subprocess.run([BIN], input='\n'.join(lines) + '\n', capture_output=True, text=True, check=True)
        return r.stdout.split()
    return run


@pytest.mark.parametrize('p', PRIMES, ids=lambda p: f'p{p.bit_length()}_{p & 0xffff:x}')
def test_field_arithmetic_on_device(checker, p):
    lines, want, (L, k) = commands(p, lazy_sizes=(1, 2, 3, 7, 17, 64))
    out = checker(lines)
    kind, Lr, kr = (int(x) for x in out[:3])
    assert (kind, Lr, kr) == (expected_kind(p), L, k)
    got = out[3:]
    assert len(got) == len(want)
    bad = [(lines[i + 1][:120], got[i], f'{want[i]:x}') for i in range(len(want)) if got[i] not in (f'{want[i]:x}', 'n/a')]
    assert not bad, bad[:5]
