"""MPyC program for K14: mpc.np_matmul of a SecInt(32) matrix with an int64 matrix on each side and with an int64 vector,
np_argmax / np_argmin along an axis and np_unit_vector (whose `u @ np.arange(n)` multiplies by a public integer vector,
runtime.py:3750-3757, 5016), a SecFxp product with a public float matrix on the left (np_matmul rounds it to an object
array of ints, runtime.py:2498-2511), and np.matmul of two field arrays opened with output(raw=True); then output.

    python tests/run_installed.py tests/programs/resident_matmul_int.py [-M3]

Prints the results, then one line per call with the engine's conversion counters around it (absent without the engine):
'counts <name> {...}', where 'matmul_settles' counts the limb-backed values turned into Python ints by the reference's
own FiniteFieldArray.__matmul__ / __rmatmul__ / __array_ufunc__ (finfields.py:728-764, 1126-1146) and 'inner_settles'
the one-element results of 1-D @ 1-D products settled by mpyc_b200.resident.matmul.
"""
import json
import sys

import numpy as np
from mpyc.runtime import mpc

settles = {'matmul': 0, 'inner': 0}


def counters():
    try:
        from mpyc_b200 import resident
    except ImportError:
        return None
    return dict(resident.calls, matmul_settles=settles['matmul'], inner_settles=settles['inner'])


def watch_matmul():
    """Count materialisations whose call stack passes through the reference's matmul methods, and those of resident.matmul."""
    try:
        from mpyc_b200 import resident
    except ImportError:
        return
    orig = resident.LimbValue._materialise

    def mat(self):
        if self._ints is None:
            f = sys._getframe(1)
            while f is not None:
                name, file = f.f_code.co_name, f.f_code.co_filename
                if name in ('__matmul__', '__rmatmul__', '__array_ufunc__') and file.endswith('finfields.py'):
                    settles['matmul'] += 1
                    break
                if name == 'matmul' and file.endswith('resident.py'):
                    settles['inner'] += 1
                    break
                f = f.f_back
        return orig(self)
    resident.LimbValue._materialise = mat


def delta(before, after):
    return None if after is None else {k: after[k] - before[k] for k in after}


async def main():
    watch_matmul()
    secint = mpc.SecInt(32)
    secfxp = mpc.SecFxp(32)
    await mpc.start()
    rng = np.random.default_rng(11)
    a = rng.integers(-1000, 1000, size=(6, 40))
    x = mpc.input(secint.array(a), senders=0)
    y = mpc.input(secfxp.array(rng.integers(-50, 50, size=(3, 4)) / 4), senders=0)
    i = mpc.input(secint(3), senders=0)
    await mpc.gather(x, y, i)
    W = rng.integers(-2**31, 2**31, size=(40, 5))
    V = rng.integers(-2**40, 2**40, size=(3, 6))
    v = rng.integers(0, 2**20, size=40).astype(np.uint32)
    X = await mpc.output(x, raw=True)
    Z = await mpc.output(mpc.np_transpose(x), raw=True)
    calls = [('matmul_xW', lambda: mpc.np_matmul(x, W)),
             ('matmul_Wx', lambda: mpc.np_matmul(V, x)),
             ('matmul_xv', lambda: mpc.np_matmul(x, v)),
             ('argmax', lambda: mpc.np_argmax(x, axis=1)),
             ('argmin', lambda: mpc.np_argmin(x, axis=0)),
             ('unit_vector', lambda: mpc.np_unit_vector(i, 8)),
             ('fxp_float_left', lambda: mpc.np_matmul(np.array([[0.5, 1.5, -2.0]]), y)),
             ('np_matmul_opened', lambda: np.matmul(X, Z))]
    results, counts = [], {}
    for name, fn in calls:
        before = counters()
        r = fn()
        if name != 'np_matmul_opened':
            r = await mpc.output(r)
        counts[name] = delta(before, counters())
        results.append((name, r))

    for name, r in results:
        v = r.value if hasattr(r, 'value') else r
        print(name, np.asarray(v).tolist())
    if counts['argmax'] is not None:
        for name, cnt in counts.items():
            print('counts', name, json.dumps(cnt))
    await mpc.shutdown()

mpc.run(main())
