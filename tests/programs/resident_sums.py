"""MPyC program for the sums of secure arrays: np_sum over several axes (with keepdims and initial), np_cumsum,
np_cumulative_sum and np_outer on products of secure integer arrays over a 128-bit prime, then output.

    python tests/run_installed.py tests/programs/resident_sums.py [-M3]

Prints the opened results, then one line 'between {...}' with the engine's conversion counters between the arrival of
the inputs and output (absent without the engine).  Under install(resident=True) every sum runs on the limbs: the
counters must show no materialised and no packed array.
"""
import json

import numpy as np
from mpyc.runtime import mpc

P128 = 2**128 - 173


def counters():
    try:
        from mpyc_b200 import resident
    except ImportError:
        return None
    return dict(resident.calls)


async def main():
    secint = mpc.SecInt(32, p=P128)
    await mpc.start()
    rng = np.random.default_rng(11)
    a = rng.integers(-2**15, 2**15, size=(3, 4, 5))
    b = rng.integers(-2**15, 2**15, size=(3, 4, 5))
    u0 = rng.integers(-2**15, 2**15, size=7)
    v0 = rng.integers(-2**15, 2**15, size=6)
    x = mpc.input(secint.array(a), senders=0)
    y = mpc.input(secint.array(b), senders=0)
    u = mpc.input(secint.array(u0), senders=0)
    v = mpc.input(secint.array(v0), senders=0)
    await mpc.gather(x, y, u, v)
    before = counters()
    z = x * y                                    # limb-backed shares after _reshare
    uu, vv = u * u, v * u[:6]
    results = [
        ('sum all', mpc.np_sum(z)),
        ('sum axis=1', mpc.np_sum(z, axis=1)),
        ('sum axis=-1 keepdims', mpc.np_sum(z, axis=-1, keepdims=True)),
        ('sum axis=(0,2) initial=5', mpc.np_sum(z, axis=(0, 2), initial=5)),
        ('sum axis=(1,2)', mpc.np_sum(z, axis=(1, 2))),
        ('sum all keepdims initial=-3', mpc.np_sum(z, keepdims=True, initial=-3)),
        ('cumsum', mpc.np_cumsum(z)),
        ('cumsum axis=1', mpc.np_cumsum(z, axis=1)),
        ('cumulative_sum axis=2', mpc.np_cumulative_sum(z, axis=2)),
        ('cumulative_sum axis=0 include_initial', mpc.np_cumulative_sum(z, axis=0, include_initial=True)),
        ('cumulative_sum 1-D include_initial', mpc.np_cumulative_sum(uu, include_initial=True)),
        ('outer', mpc.np_outer(uu, vv)),
    ]
    await mpc.gather(*[r for _, r in results])
    after = counters()
    for name, r in results:
        got = await mpc.output(r)
        print(name, np.shape(got), np.asarray(got).reshape(-1).tolist())
    if after is not None:
        print('between', json.dumps({k: after[k] - before[k] for k in after}))
    await mpc.shutdown()

mpc.run(main())
