"""MPyC program for the protocols that move secure arrays around between their GPU steps: np_sort along an axis,
np_argmax, np_amax, np_add_bits and a 2 x 2 max-pooling of image-shaped arrays with strided selections (as in the
reference's np_cnnmnist demo), on products of secure integer arrays over a 128-bit prime, then output.

    python tests/run_installed.py tests/programs/resident_protocols.py [-M3]

Prints the opened results, then one line 'between {...}' with the engine's conversion counters between the arrival of
the inputs and output (absent without the engine).
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


def maxpool(x):
    x = mpc.np_maximum(x[:, :, ::2, :], x[:, :, 1::2, :])
    return mpc.np_maximum(x[:, :, :, ::2], x[:, :, :, 1::2])


async def main():
    secint = mpc.SecInt(32, p=P128)
    secbits = mpc.SecInt(2, p=P128)
    await mpc.start()
    rng = np.random.default_rng(13)
    a = rng.integers(-2**10, 2**10, size=(3, 6))
    m = rng.integers(-2**10, 2**10, size=(1, 2, 4, 4))
    bits_a = rng.integers(0, 2, size=(2, 5))
    bits_b = rng.integers(0, 2, size=(2, 5))
    x = mpc.input(secint.array(a), senders=0)
    img = mpc.input(secint.array(m), senders=0)
    ba = mpc.input(secbits.array(bits_a), senders=0)
    bb = mpc.input(secbits.array(bits_b), senders=0)
    await mpc.gather(x, img, ba, bb)
    before = counters()
    z = x * x - x                                # limb-backed shares after _reshare
    im = img * img
    results = [
        ('sort axis=1', mpc.np_sort(z, axis=1)),
        ('argmax axis=0', mpc.np_argmax(z, axis=0)),
        ('amax', mpc.np_amax(z)),
        ('add_bits', mpc.np_add_bits(ba * ba, bb * bb)),
        ('maxpool', maxpool(im)),
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
