"""MPyC program for the layout of secure arrays: selections with steps, negative steps, None and an index array,
transposes, joins, flips, rolls, a broadcast product and writes through a slice and an index array, on products of secure
integer arrays over a 128-bit prime, then output.

    python tests/run_installed.py tests/programs/resident_layout.py [-M3]

Prints the opened results, then one line 'between {...}' with the engine's conversion counters between the arrival of
the inputs and output (absent without the engine).  Under install(resident=True) every step runs on the limbs: the
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
    rng = np.random.default_rng(12)
    a = rng.integers(-2**15, 2**15, size=(4, 6))
    b = rng.integers(-2**15, 2**15, size=(4, 6))
    c = rng.integers(-2**15, 2**15, size=(2, 3, 4))
    x = mpc.input(secint.array(a), senders=0)
    y = mpc.input(secint.array(b), senders=0)
    w = mpc.input(secint.array(c), senders=0)
    await mpc.gather(x, y, w)
    before = counters()
    z = x * y                                    # limb-backed shares after _reshare
    z2 = y * y
    t = w * w
    u1, u2 = x * z2, z2 * y                      # written to once each (np_update changes the reference's array in place)
    results = [
        ('getitem steps', z[:, ::2]),
        ('getitem negative step', z[::-1, 1::3]),
        ('getitem None', z[None, 1, :, None]),
        ('getitem index array', z[:, [5, 0, 2]]),
        ('transpose axes', mpc.np_transpose(t, axes=(2, 0, 1))),
        ('swapaxes', mpc.np_swapaxes(t, 0, 2)),
        ('concatenate axis=1', mpc.np_concatenate((z, z2), axis=1)),
        ('concatenate axis=-1', mpc.np_concatenate((t, t[:, :, :1]), axis=-1)),
        ('concatenate axis=None', mpc.np_concatenate((z, t), axis=None)),
        ('stack axis=1', mpc.np_stack((z, z2), axis=1)),
        ('vstack', mpc.np_vstack((z, z2[0]))),
        ('hstack', mpc.np_hstack((z, z2[:, :2]))),
        ('flip', mpc.np_flip(t, axis=(0, 2))),
        ('roll', mpc.np_roll(z, 2, axis=1)),
        ('broadcast multiply', mpc.np_multiply(z[:, :1], z2)),
        ('update slice', mpc.np_update(u1, (slice(1, 3),), z2[:2])),
        ('update index array', mpc.np_update(u2, (Ellipsis, [4, 1]), z[:, :2])),
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
