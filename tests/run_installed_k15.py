"""Launcher: tests/run_installed.py with install(public_matmul=True) and, in 'oracle' mode, K7's to K15's stand-ins
(tests/oracle_reduce.py, tests/oracle_layout.py, tests/oracle_linalg.py, tests/oracle_conv.py, tests/oracle_divsel.py,
tests/oracle_powexp.py, tests/oracle_prod.py, tests/oracle_matmul_int.py, tests/oracle_gf.py) added to the CPU oracle
backend, so that GF(2^8) broadcasts, stacked products and bit compositions take mpyc_b200.resident's device path as they do
on a GPU.  Same
arguments and environment as run_installed.py; MPyC's -M re-execution runs every party through this launcher."""
import functools
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(HERE), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

if __name__ == '__main__':
    flags = os.environ.get('MPYC_B200_HARNESS', 'install').split(',')
    if 'off' not in flags:
        import mpyc_b200.install as inst
        inst.install = functools.partial(inst.install, public_matmul=True)
    if 'oracle' in flags:
        import oracle_conv
        import oracle_device
        import oracle_divsel
        import oracle_gf
        import oracle_layout
        import oracle_linalg
        import oracle_matmul_int
        import oracle_powexp
        import oracle_prod
        import oracle_reduce
        for m in (oracle_reduce, oracle_layout, oracle_linalg, oracle_conv, oracle_divsel, oracle_powexp, oracle_prod,
                  oracle_matmul_int, oracle_gf):
            m.extend(oracle_device.OracleBackend)
    runpy.run_path(os.path.join(HERE, 'run_installed.py'), run_name='__main__')
