"""MPyC program for secret exponents: 2 ** x and mpc.np_pow(3, x) of SecInt(32) arrays, mpc.np_exp2 and mpc.np_exp of
SecFxp(32) arrays, and np_pow(2, x) over GF(2^128 - 173) -- every one of them Runtime._np_pow_public_int_base_secret_
integral_exponent, whose two gmpy.powmod_exp_list calls (runtime.py:1408,1422) are the exponentiations K12 takes over --
then output.  With more than one party the integral exponents are SecFxp(32) arrays (see below).

    python tests/run_installed.py tests/programs/resident_powexp.py [-M3]

Prints the results, then one line per call with the engine's conversion counters around it, from the call to its
gathered result (absent without the engine): 'counts <name> {...}', and 'lists <name> <n>' with the number of
gmpy.powmod_exp_list calls the protocol made.
"""
import json

import numpy as np
from mpyc import gmpy
from mpyc.runtime import mpc


def counters():
    try:
        from mpyc_b200 import resident
    except ImportError:
        return None
    return dict(resident.calls)


def delta(before, after):
    return None if after is None else {k: after[k] - before[k] for k in after}


lists = [0]


def counted(fn):
    def call(*args):
        lists[0] += 1
        return fn(*args)
    return call


async def main():
    gmpy.powmod_exp_list = counted(gmpy.powmod_exp_list)      # whatever install() put there: count the protocol's calls
    secfxp = mpc.SecFxp(32)
    if len(mpc.parties) == 1:
        secint, secint128 = mpc.SecInt(32), mpc.SecInt(32, p=2**128 - 173)
    else:
        # the reference's protocol builds SecureIntegerArray(shape=..., integral=True) on the parties that draw no r
        # (runtime.py:1412), which that class does not accept: with several parties its integral exponents are SecFxp
        secint, secint128 = secfxp, mpc.SecFxp(32, p=2**128 - 173)
    await mpc.start()
    n = 200
    rng = np.random.default_rng(5)
    e = rng.integers(0, 31, size=n)
    f = rng.integers(0, 20, size=n)
    g = rng.uniform(-4, 4, size=16).round(3)
    x = mpc.input(secint.array(e), senders=0)
    y = mpc.input(secint.array(f), senders=0)
    u = mpc.input(secfxp.array(g), senders=0)
    z = mpc.input(secint128.array(e), senders=0)
    for v in (x, y, z):
        if secint is secfxp:
            v.integral = True
    await mpc.gather(x, y, u, z)

    calls = [('pow2', lambda: 2 ** x), ('np_pow3', lambda: mpc.np_pow(3, y)), ('exp2', lambda: mpc.np_exp2(u)),
             ('exp', lambda: mpc.np_exp(u)), ('pow2_p128', lambda: mpc.np_pow(2, z))]
    results, counts, nlists = [], {}, {}
    for name, fn in calls:
        before, l0 = counters(), lists[0]
        r = fn()
        await mpc.gather(r)
        counts[name] = delta(before, counters())
        nlists[name] = lists[0] - l0
        results.append((name, r))

    for name, r in results:
        v = await mpc.output(r)
        v = np.asarray(v)
        print(name, (v.round(2) if v.dtype.kind == 'f' else v).tolist())
    for name in nlists:
        print('lists', name, nlists[name])
    if counts['pow2'] is not None:
        for name, cnt in counts.items():
            print('counts', name, json.dumps(cnt))
    await mpc.shutdown()

mpc.run(main())
