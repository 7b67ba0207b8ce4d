"""MPyC program for secure convolutions: Runtime.np_convolve of secure integer arrays in all three modes and both length
orders, with a public integer array, of secure fixed-point arrays (with each other, and with a public float array in
'same' mode) and of secure prime-field arrays; Runtime.np_roll by a secret shift, whose local step convolves with a
secret unit vector; one secure polynomial product and one divmod (mpyc.secpols, built from np_convolve and np_roll),
then output.

    python tests/run_installed.py tests/programs/resident_conv.py [-M3]

Prints the results, then two lines with the engine's conversion counters (absent without the engine):
  'counts conv {...}'  around the np_convolve calls: under install(resident=True) the gathered shares are convolved on
                       their limbs, so the counters must show no materialised array and one packed array per public
                       operand;
  'counts roll {...}'  around the np_roll call: no materialised array, and the one pack of np_fromlist's unit vector.
"""
import json

import numpy as np
from mpyc.runtime import mpc
from mpyc.secpols import secpoly


def counters():
    try:
        from mpyc_b200 import resident
    except ImportError:
        return None
    return dict(resident.calls)


def delta(before, after):
    return None if after is None else {k: after[k] - before[k] for k in after}


async def main():
    secint = mpc.SecInt(32)
    secfxp = mpc.SecFxp(32)
    secfld = mpc.SecFld(2**61 - 1)
    await mpc.start()
    rng = np.random.default_rng(7)
    a = rng.integers(-2**10, 2**10, size=9)
    b = rng.integers(-2**10, 2**10, size=5)
    c = rng.integers(-2**10, 2**10, size=4)
    x = mpc.input(secint.array(a), senders=0)
    y = mpc.input(secint.array(b), senders=0)
    u = mpc.input(secfxp.array(np.array([0.5, -1.25, 2.0, 3.5, -0.75])), senders=0)
    v = mpc.input(secfxp.array(np.array([1.5, 0.25, -2.0])), senders=0)
    f = mpc.input(secfld.array(np.array([3, 1, 4, 1, 5, 9, 2, 6])), senders=0)
    g = mpc.input(secfld.array(np.array([2, 7, 1])), senders=0)
    s = mpc.input(secint(3), senders=0)
    await mpc.gather(x, y, u, v, f, g, s)

    before = counters()
    results = []
    for mode in ('full', 'same', 'valid'):
        results.append((f'int {mode}', mpc.np_convolve(x, y, mode=mode)))
        results.append((f'int swapped {mode}', mpc.np_convolve(y, x, mode=mode)))
    results.append(('int public', mpc.np_convolve(x, c)))
    results.append(('fxp', mpc.np_convolve(u, v)))
    results.append(('fxp public same', mpc.np_convolve(u, np.array([0.5, -1.5, 2.25]), mode='same')))
    results.append(('fld', mpc.np_convolve(f, g)))
    await mpc.gather([r for _, r in results])          # the shares: every convolution has run
    conv_counts = delta(before, counters())

    before = counters()
    rolled = mpc.np_roll(x, s)
    await mpc.gather(rolled)
    roll_counts = delta(before, counters())

    p = secpoly(secfld.array(np.array([1, 2, 3, 4])))
    q = secpoly(secfld.array(np.array([5, 0, 6])))
    product = p * q
    quotient, remainder = divmod(p, q)

    for name, r in results:
        print(name, np.asarray(await mpc.output(r)).tolist())
    print('roll', np.asarray(await mpc.output(rolled)).tolist())
    for name, poly in (('poly product', product), ('poly quotient', quotient), ('poly remainder', remainder)):
        print(name, await mpc.output(poly))
    if conv_counts is not None:
        print('counts conv', json.dumps(conv_counts))
        print('counts roll', json.dumps(roll_counts))
    await mpc.shutdown()

mpc.run(main())
