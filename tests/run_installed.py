"""Launcher: run an UNMODIFIED MPyC program (a demo of the reference, or any script using `from mpyc.runtime import mpc`)
with the GPU engine installed behind mpyc.thresha / mpyc.finfields.

    python tests/run_installed.py <program.py> [program and MPyC flags, e.g. -M3 -1]

MPyC's multi-party mode re-executes sys.argv for the other parties (mpyc/runtime.py:5156-5189), so every party goes
through this launcher and gets the same installation.  Configuration travels in the environment so that it reaches
the child parties too:
    MPYC_REFERENCE           path of the reference checkout / install (prepended to sys.path); default: importable mpyc
    MPYC_B200_HARNESS        comma list: install (default), oracle (no GPU: device round trips answered by
                             tests/oracle_device.py -- test infrastructure), limb_wire, finfields, ops (operator hooks),
                             resident (limb-resident arrays), spread (party i on GPU i mod #GPUs), verify (real device calls, every
                             result cross-checked against the oracle; mismatches logged and raised), strict, off
    MPYC_B200_OPS_MIN_SIZE   install(operators_min_size=...)
    MPYC_B200_MIN_SIZE       install(min_size=...)
    MPYC_B200_FORCE_PRIME    hex prime: SecInt/SecFxp types are built over this prime (BASELINE configs[4]: 256-bit)
    MPYC_B200_CALL_LOG       file: one line per engine call (name, field bits, elements), appended per process
    MPYC_B200_STATS          1: print mpyc_b200.resident.calls (limb ops, materialisations, packs, ModValues) at exit
"""
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
sys.dont_write_bytecode = True
ref = os.environ.get('MPYC_REFERENCE')
if ref:
    sys.path.insert(0, ref)


def main():
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    flags = set(filter(None, os.environ.get('MPYC_B200_HARNESS', 'install').split(',')))
    from mpyc.runtime import mpc   # noqa: F401  (parses sys.argv, spawns the other parties with this launcher)
    import mpyc.thresha
    import mpyc.finfields
    if 'off' not in flags:
        import mpyc_b200.install as inst
        if 'oracle' in flags:
            import oracle_device
            oracle_device.patch()
            oracle_device.patch_finfields()
            oracle_device.patch_resident()
        if 'verify' in flags:            # real device calls, each result cross-checked against the oracle
            import oracle_device
            oracle_device.verify(os.environ.get('MPYC_B200_VERIFY_LOG', '/tmp/mpyc_b200_verify.log'))
        kwargs = {'strict': 'strict' in flags, 'limb_wire': 'limb_wire' in flags,
                  'min_size': int(os.environ.get('MPYC_B200_MIN_SIZE', '0'))}
        if 'finfields' in flags or 'ops' in flags:
            kwargs['finfields_module'] = mpyc.finfields
        if 'ops' in flags or 'resident' in flags:
            kwargs['operators'] = True
            kwargs['operators_min_size'] = int(os.environ.get('MPYC_B200_OPS_MIN_SIZE', '1024'))
        if 'resident' in flags:
            kwargs['resident'] = True
            kwargs['finfields_module'] = mpyc.finfields
        if os.environ.get('MPYC_B200_DEVICE'):
            kwargs['device'] = int(os.environ['MPYC_B200_DEVICE'])
        elif 'spread' in flags:           # co-located parties: party i on GPU i mod #GPUs
            import mpyc_b200
            import ctypes
            cnt = ctypes.c_int(0)
            mpyc_b200._cabi.lib.mpyc_b200_device_count(ctypes.byref(cnt))
            kwargs['device'] = mpc.pid % max(cnt.value, 1)
        inst.install(mpyc.thresha, **kwargs)
        log = os.environ.get('MPYC_B200_CALL_LOG')
        if log:
            _log_calls(mpyc.thresha, log)
    prime = os.environ.get('MPYC_B200_FORCE_PRIME')
    if prime:
        _force_prime(mpc, int(prime, 16))
    program = sys.argv[1]
    sys.argv = [program] + sys.argv[2:]
    if os.environ.get('MPYC_B200_STATS'):          # conversion / limb-op counters of this party on stderr at exit
        import atexit
        import json

        sites = {}
        if os.environ['MPYC_B200_STATS'] == 'sites':     # where limb-backed values become Python ints / get packed
            from mpyc_b200 import resident, codec

            def caller():
                f = sys._getframe(2)
                while f is not None and ('mpyc_b200' in f.f_code.co_filename or 'numpy' in f.f_code.co_filename):
                    f = f.f_back
                return f'{os.path.basename(f.f_code.co_filename)}:{f.f_code.co_name}:{f.f_lineno}' if f else '?'
            orig_mat = resident.LimbValue._materialise

            def mat(self):
                if self._ints is None:
                    key = 'materialise ' + caller()
                    sites[key] = sites.get(key, 0) + 1
                return orig_mat(self)
            resident.LimbValue._materialise = mat
            orig_pack = codec.ints_to_limbs

            def pack(values, ctx, reduce=True):
                key = 'pack ' + caller()
                sites[key] = sites.get(key, 0) + 1
                return orig_pack(values, ctx, reduce=reduce)
            codec.ints_to_limbs = pack

        def _stats():
            from mpyc_b200 import resident
            sys.stderr.write('MPYC_B200_STATS ' + json.dumps({'pid': mpc.pid, **resident.calls}) + '\n')
            for key, cnt in sorted(sites.items(), key=lambda kv: -kv[1])[:25]:
                sys.stderr.write(f'MPYC_B200_SITE pid={mpc.pid} {cnt:5d} {key}\n')
        atexit.register(_stats)
    runpy.run_path(program, run_name='__main__')


def _force_prime(mpc, p):
    """SecInt / SecFxp factories accept p= (mpyc/sectypes.py:685-718); the demos do not pass it."""
    for name in ('SecInt', 'SecFxp'):
        orig = getattr(mpc, name)

        def factory(*args, _orig=orig, **kwargs):
            kwargs.setdefault('p', p)
            return _orig(*args, **kwargs)
        setattr(mpc, name, factory)


def _log_calls(module, path):
    import functools
    names = ('random_split', 'recombine', 'np_random_split', 'np_recombine', 'pseudorandom_share',
             'pseudorandom_share_zero', 'np_pseudorandom_share', 'np_pseudorandom_share_0')
    fh = open(path, 'a')

    def wrap(name, fn):
        @functools.wraps(fn)
        def call(field, *args, **kwargs):
            try:
                if 'split' in name:
                    n = len(args[0])
                elif 'recombine' in name:
                    n = len(args[0][0][1])
                else:
                    n = int(args[-1])
            except Exception:   # noqa: BLE001
                n = -1
            fh.write(f'{os.getpid()} {name} {getattr(field, "order", 0).bit_length()} {n}\n')
            fh.flush()
            return fn(field, *args, **kwargs)
        return call
    for name in names:
        setattr(module, name, wrap(name, getattr(module, name)))


if __name__ == '__main__':
    main()
