"""MPyC program for secure division and selection: == and != of SecInt(64) arrays (Runtime._np_is_zero, whose np.where steps
select raw share values), Runtime.np_reciprocal and / of SecInt(32) arrays, / of SecFld(2^61 - 1) arrays, np_divide by a
public field array, np_lsb and np_from_bits, then output.

    python tests/run_installed.py tests/programs/resident_divsel.py [-M3]

Prints the results, then one line per call with the engine's conversion counters around it, from the call to its
gathered result (absent without the engine): 'counts <name> {...}'.
"""
import json

import numpy as np
from mpyc.runtime import mpc


def counters():
    try:
        from mpyc_b200 import resident
    except ImportError:
        return None
    return dict(resident.calls)


def delta(before, after):
    return None if after is None else {k: after[k] - before[k] for k in after}


async def main():
    secint64 = mpc.SecInt(64)
    secint = mpc.SecInt(32)
    secfld = mpc.SecFld(2**61 - 1)
    await mpc.start()
    n = 40
    rng = np.random.default_rng(11)
    a = rng.integers(-2**40, 2**40, size=n)
    b = np.where(rng.integers(0, 2, size=n) == 1, a, rng.integers(-2**40, 2**40, size=n))
    c = rng.integers(1, 2**20, size=n) * rng.choice([-1, 1], size=n)
    d = rng.integers(-2**20, 2**20, size=n)
    e = rng.integers(1, 2**61 - 1, size=n)
    bits = rng.integers(0, 2, size=(n, 8))
    x = mpc.input(secint64.array(a), senders=0)
    y = mpc.input(secint64.array(b), senders=0)
    u = mpc.input(secint.array(c), senders=0)
    w = mpc.input(secint.array(d), senders=0)
    f = mpc.input(secfld.array(e), senders=0)
    g = mpc.input(secfld.array(e[::-1].copy()), senders=0)
    t = mpc.input(secint.array(bits), senders=0)
    await mpc.gather(x, y, u, w, f, g, t)

    calls = [('eq', lambda: x == y), ('ne', lambda: x != y), ('reciprocal', lambda: mpc.np_reciprocal(u)),
             ('int_div', lambda: w / u), ('fld_div', lambda: f / g),
             ('public_div', lambda: mpc.np_divide(f, secfld.field.array(e[::-1].copy()))),
             ('lsb', lambda: mpc.np_lsb(u)), ('from_bits', lambda: mpc.np_from_bits(t))]
    results, counts = [], {}
    for name, fn in calls:
        before = counters()
        r = fn()
        await mpc.gather(r)
        counts[name] = delta(before, counters())
        results.append((name, r))

    for name, r in results:
        print(name, np.asarray(await mpc.output(r)).tolist())
    if counts['eq'] is not None:
        for name, cnt in counts.items():
            print('counts', name, json.dumps(cnt))
    await mpc.shutdown()

mpc.run(main())
