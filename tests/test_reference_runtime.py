"""Caller-level harness: the UNMODIFIED reference runtime (mpyc/runtime.py, sectypes.py, the demos and the reference's
own unittest files) running on top of mpyc_b200.install().

Two device modes, same tests:
  * 'oracle'  (build container, no GPU; not gpu-marked): the four device round trips of mpyc_b200.thresha are answered
    by tests/oracle_device.py, everything above them is the product code.
  * 'cuda'    (-m gpu): the real kernels through the C ABI.
Both need the reference: $MPYC_REFERENCE, or the copy of it that build() makes in oracle/_ref/ (oracle/reference.py);
they skip where it is absent.

Every run goes through tests/run_installed.py in a child process (MPyC parses sys.argv and builds its runtime at import;
-M3 re-executes the command line for the other parties, mpyc/runtime.py:5156-5189).
Pinned here: reference tests/test_thresha.py, test_finfields.py, test_runtime.py (20/20) under install(); np_aes.py
(FIPS-197 ciphertext, docs/demos.rst:606-611) and np_cnnmnist.py (logits identical to the uninstalled run), 1 party
and -M3; and tests/programs/secure_ops.py, installed == uninstalled, 1 party and -M3.
"""
import itertools
import os
import subprocess
import sys

import pytest

from oracle import reference

HERE = os.path.dirname(os.path.abspath(__file__))
LAUNCHER = os.path.join(HERE, 'run_installed.py')
PROGRAM = os.path.join(HERE, 'programs', 'secure_ops.py')
FIPS197 = '69c4e0d86a7b0430d8cdb78070b4c55a'


REF = reference.path()


def _checkout_dir(name):
    """The reference's tests/ or demos/ directory, where the reference copy has it."""
    if REF and os.path.isdir(os.path.join(REF, name)):
        return os.path.join(REF, name)
    return None


TESTS_DIR = _checkout_dir('tests')
DEMOS_DIR = _checkout_dir('demos')
HAVE_TESTS = TESTS_DIR is not None
HAVE_DEMOS = DEMOS_DIR is not None and os.path.isfile(os.path.join(DEMOS_DIR, 'np_aes.py'))
_ports = itertools.count(13000 + (os.getpid() % 400) * 40, 8)


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except ImportError:
        return False


@pytest.fixture(params=['oracle', pytest.param('cuda', marks=pytest.mark.gpu)])
def mode(request):
    if REF is None:
        pytest.skip('no reference available ($MPYC_REFERENCE or the copy build() makes in oracle/_ref)')
    if request.param == 'cuda' and not _has_cuda():
        pytest.skip('no CUDA device')
    if request.param == 'oracle' and _has_cuda():
        pytest.skip('GPU present: the cuda variant runs the real kernels instead of the oracle stand-in')
    return request.param


def trim_for_gpu(mode, keep):
    """The cuda variants run a subset (the driver's GPU test slot is minutes, and every run pays interpreter start + CUDA
    context creation per party): multi-party runs and the most invasive configurations.  MPYC_B200_FULL_GPU_HARNESS=1
    runs everything."""
    if mode == 'cuda' and not keep and os.environ.get('MPYC_B200_FULL_GPU_HARNESS') != '1':
        pytest.skip('not in the GPU subset (MPYC_B200_FULL_GPU_HARNESS=1 runs it)')


def run(mode, program, args=(), flags=('install',), cwd=None, timeout=900, parties=1, env_extra=None):
    flags = list(flags)
    if mode == 'oracle' and 'off' not in flags:
        flags.append('oracle')
    env = dict(os.environ, MPYC_REFERENCE=REF, MPYC_B200_HARNESS=','.join(flags), PYTHONDONTWRITEBYTECODE='1')
    env.update(env_extra or {})
    cmd = [sys.executable, LAUNCHER, program, *args, '--no-log']
    if parties > 1:
        cmd += [f'-M{parties}', '-B', str(next(_ports))]
    r = subprocess.run(cmd, cwd=cwd or HERE, env=env, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, f'{cmd} failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}'
    return r.stdout


WIDER = ('test_sectypes', 'test_secpols', 'test_statistics', 'test_asyncoro', 'test_fingroups', 'test_gfpx', 'test_gmpy',
         'test_mpctools', 'test_numpy', 'test_random', 'test_secgroups', 'test_seclists')    # + thresha, finfields, runtime: all 84 tests
EVERYTHING = {'MPYC_B200_OPS_MIN_SIZE': '1'}    # every array operator call goes through the hooks, whatever its size


@pytest.mark.parametrize('flags', [('install',), ('install', 'limb_wire'), ('install', 'ops'), ('install', 'resident')],
                         ids=lambda f: '+'.join(f))
@pytest.mark.parametrize('name', ['test_thresha', 'test_finfields', 'test_runtime', *WIDER])
def test_reference_unittests_under_install(mode, name, flags):
    """The reference's own unit tests, all green with the engine behind mpyc.thresha (and, with 'ops' / 'resident', behind
    the FiniteFieldArray operators, the batched inverse/pow/sqrt and the limb-resident `.value`, with the size
    threshold at 1 so that every operator call takes the hooked path)."""
    if not HAVE_TESTS:
        pytest.skip('reference tests/ directory not available (package-only reference)')
    if name in WIDER and flags != ('install', 'resident'):
        pytest.skip('the wider suites run once, in the most invasive configuration')
    trim_for_gpu(mode, flags in (('install',), ('install', 'resident')) and name in ('test_thresha', 'test_finfields', 'test_runtime', 'test_secpols'))
    out = run(mode, os.path.join(HERE, 'ref_unittest.py'), [os.path.join(TESTS_DIR, name + '.py')], flags,
              env_extra=EVERYTHING)
    assert 'failures=0 errors=0' in out, out[-2000:]
    if name == 'test_runtime':
        assert 'REFTESTS run=20 ' in out


@pytest.mark.parametrize('flags', [('install',), ('install', 'resident')], ids=lambda f: '+'.join(f))
@pytest.mark.parametrize('parties', [1, 3])
def test_np_aes_fips197(mode, parties, flags):
    """BASELINE configs[3]: demos/np_aes.py unchanged; AES-128 of the FIPS-197 example block."""
    if not HAVE_DEMOS:
        pytest.skip('reference demos/ not available (package-only reference)')
    trim_for_gpu(mode, parties == 3)
    out = run(mode, 'np_aes.py', ['-1'], flags, cwd=DEMOS_DIR, parties=parties, env_extra=EVERYTHING)
    assert f'Ciphertext:  {FIPS197}' in out, out


@pytest.mark.parametrize('parties', [1, 3])
def test_np_cnnmnist_logits_identical(mode, parties):
    """demos/np_cnnmnist.py unchanged (one image, offset 0): prediction and the 10 opened logits identical to the run
    without the engine."""
    if not HAVE_DEMOS:
        pytest.skip('reference demos/ not available (package-only reference)')
    cwd = DEMOS_DIR
    trim_for_gpu(mode, parties == 3)
    if mode == 'oracle' and parties == 3 and os.environ.get('MPYC_B200_FULL_CPU_HARNESS') != '1':
        pytest.skip('45 s of Python modular exponentiations in the oracle stand-in; the -M3 run is covered with the real kernels '
                    '(-m gpu) and by the 1-party oracle run (MPYC_B200_FULL_CPU_HARNESS=1 runs it here too)')
    want = run(mode, 'np_cnnmnist.py', ['1', '0'], ('off',), cwd=cwd, parties=parties)
    got = run(mode, 'np_cnnmnist.py', ['1', '0'], ('install', 'resident'), cwd=cwd, parties=parties,
              env_extra={'MPYC_B200_OPS_MIN_SIZE': '64'})
    tail = lambda s: s[s.index('Image #0'):]   # noqa: E731
    assert 'with label 7: 7 predicted' in got
    assert tail(got) == tail(want)


@pytest.mark.parametrize('flags', [('install',), ('install', 'resident')], ids=lambda f: '+'.join(f))
@pytest.mark.parametrize('parties', [1, 3])
def test_secure_ops_program_installed_equals_reference(mode, parties, flags):
    """tests/programs/secure_ops.py (input, output, multiply, matmul, comparisons, random bits, fixed-point truncation,
    convert, GF(2^8) inversion, field division): opened results identical with and without the engine."""
    trim_for_gpu(mode, parties == 3)
    want = run(mode, PROGRAM, ['48'], ('off',), parties=parties)
    got = run(mode, PROGRAM, ['48'], flags, parties=parties, env_extra=EVERYTHING)
    assert 'field division' in got
    assert got == want


@pytest.mark.parametrize('parties', [1, 3])
def test_conv_layer_bound_to_the_engine_equals_the_object_loops(mode, parties):
    """tests/programs/cnn_conv.py: a secure convolution layer written like the CNN demo's (gather, correlate on raw values,
    field.array, _reshare) with the local step bound to mpyc_b200.resident.conv2d (K6 k_conv2d) -- INTEGRATION.md
    section 5 -- against the same program running its NumPy object loops on the plain reference."""
    trim_for_gpu(mode, parties == 3)
    want = run(mode, os.path.join(HERE, 'programs', 'cnn_conv.py'), ['2'], ('off',), parties=parties)
    got = run(mode, os.path.join(HERE, 'programs', 'cnn_conv.py'), ['2'], ('install', 'resident'), parties=parties,
              env_extra=EVERYTHING)
    assert got.count('digest=') == 2 and got == want


@pytest.mark.parametrize('parties', [1, 3])
def test_local_algebra_of_protocols_runs_on_limbs(mode, parties):
    """Secure comparisons, random bits and fixed-point products (np_sgn, np_random_bits, np_trunc) with
    install(resident=True): the whitelisted protocol functions receive ModValues (their raw-value algebra runs mod p on the
    K1 / K6 kernels), and the opened results equal the plain reference's."""
    import json
    trim_for_gpu(mode, parties == 3)
    want = run(mode, PROGRAM, ['300'], ('off',), parties=parties)
    out = subprocess.run([sys.executable, LAUNCHER, PROGRAM, '300', '--no-log'] + ([f'-M{parties}', '-B', str(next(_ports))] if parties > 1 else []),
                         cwd=HERE, capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, MPYC_REFERENCE=REF, PYTHONDONTWRITEBYTECODE='1', MPYC_B200_STATS='1', MPYC_B200_OPS_MIN_SIZE='64',
                                  MPYC_B200_HARNESS='install,resident' + (',oracle' if mode == 'oracle' else '')))
    assert out.returncode == 0, out.stderr[-3000:]
    assert out.stdout == want
    stats = [json.loads(line.split(' ', 1)[1]) for line in out.stderr.splitlines() if line.startswith('MPYC_B200_STATS ')]
    mine = [s for s in stats if s['pid'] == 0]
    assert mine and mine[0]['mod_values'] >= 10 and mine[0]['limb_ops'] >= 30


@pytest.mark.parametrize('parties', [1, 3])
def test_resident_chain_creates_no_python_ints_between_input_and_output(mode, parties):
    """input -> a*b -> _reshare -> (a*b)*a -> _reshare -> output over a 128-bit prime with install(resident=True):
    the product code performs no int <-> limb conversion between the arrival of the input shares and output()
    (and on a GPU box the C codec is not called at all in between); result equal to NumPy's."""
    import json
    out = run(mode, os.path.join(HERE, 'programs', 'resident_chain.py'), ['3000'], ('install', 'resident'), parties=parties)
    rec = json.loads(out.strip().splitlines()[-1])
    assert rec['ok'] and rec['n'] == 3000 and rec['parties'] == parties
    between = rec['conversions_between']
    assert between['materialised'] == 0 and between['packed'] == 0
    assert between['limb_ops'] == 2                      # the two local products ran on limbs
    if mode == 'cuda':
        assert between['pycodec'] == 0                   # (the oracle stand-in converts internally; the kernels do not)
