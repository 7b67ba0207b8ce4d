"""MPyC program for K13: mpc.np_is_zero_public and x < y of SecInt(16) arrays (a 48-bit field, so np_is_zero_public takes
its small-field branch and tests `np.all(await self.output(rs, ...))`, runtime.py:965), then np.prod, np.cumprod, np.all and
np.any of field arrays opened with output(raw=True), then output.

    python tests/run_installed.py tests/programs/resident_prod.py [-M3]

Prints the results, then one line per call with the engine's conversion counters around it (absent without the engine):
'counts <name> {...}', where 'zero_test_settles' counts the limb-backed values turned into Python ints inside
Runtime.np_is_zero_public.
"""
import json
import sys

import numpy as np
from mpyc.runtime import mpc

settles_in_zero_test = [0]


def counters():
    try:
        from mpyc_b200 import resident
    except ImportError:
        return None
    return dict(resident.calls, zero_test_settles=settles_in_zero_test[0])


def watch_zero_test():
    """Count materialisations whose call stack passes through Runtime.np_is_zero_public."""
    try:
        from mpyc_b200 import resident
    except ImportError:
        return
    orig = resident.LimbValue._materialise

    def mat(self):
        if self._ints is None:
            f = sys._getframe(1)
            while f is not None:
                if f.f_code.co_name == 'np_is_zero_public' and f.f_code.co_filename.endswith('runtime.py'):
                    settles_in_zero_test[0] += 1
                    break
                f = f.f_back
        return orig(self)
    resident.LimbValue._materialise = mat


def delta(before, after):
    return None if after is None else {k: after[k] - before[k] for k in after}


async def main():
    watch_zero_test()
    secint = mpc.SecInt(16)
    await mpc.start()
    rng = np.random.default_rng(7)
    a = rng.integers(-500, 500, size=(6, 40))
    b = rng.integers(-500, 500, size=(6, 40))
    b[0, :5] = a[0, :5]
    a[2, 7] = 0
    x = mpc.input(secint.array(a), senders=0)
    y = mpc.input(secint.array(b), senders=0)
    await mpc.gather(x, y)

    X = await mpc.output(x, raw=True)
    Y = await mpc.output(y, raw=True)
    calls = [('is_zero_public', lambda: mpc.np_is_zero_public(x - y)),
             ('lt', lambda: x < y),
             ('prod', lambda: np.prod(X, axis=1)),
             ('prod_all', lambda: np.prod(Y)),
             ('prod_method', lambda: X.prod(axis=0, keepdims=True)),
             ('cumprod', lambda: np.cumprod(X, axis=1)),
             ('cumulative_prod', lambda: np.cumulative_prod(Y, axis=0, include_initial=True)),
             ('all', lambda: np.all(X, axis=1)),
             ('any', lambda: np.any(X - Y, axis=(0, 1))),
             ('all_none', lambda: np.all(X)),
             ('any_none', lambda: np.any(X - X))]
    results, counts = [], {}
    for name, fn in calls:
        before = counters()
        r = fn()
        if name == 'is_zero_public':
            r = await r
        elif name == 'lt':
            await mpc.gather(r)
        counts[name] = delta(before, counters())
        results.append((name, r))

    for name, r in results:
        if name == 'lt':
            r = await mpc.output(r)
        if name in ('all_none', 'any_none'):
            print(name, type(r).__name__, bool(r))
            continue
        v = r.value if hasattr(r, 'value') else r
        print(name, np.asarray(v).tolist() if isinstance(v, np.ndarray) else int(v))
    if counts['prod'] is not None:
        for name, cnt in counts.items():
            print('counts', name, json.dumps(cnt))
    await mpc.shutdown()

mpc.run(main())
