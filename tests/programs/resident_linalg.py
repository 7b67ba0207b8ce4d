"""MPyC program for linear algebra over a 128-bit prime: the secure determinant Runtime.np_det (which opens L @ (U @ A) and
takes np.linalg.det of the opened array), then np.linalg.det / solve / inv / matrix_power of opened products of secure
integer arrays, then output.

    python tests/run_installed.py tests/programs/resident_linalg.py [-M3]

Prints the results, then two lines with the engine's conversion counters (absent without the engine):
  'counts public {...}'  around the public np.linalg calls on the opened arrays: under install(resident=True) they run
                         on the limbs, so the counters must show no materialised and no packed array;
  'counts np_det {...}'  around the whole mpc.np_det call, the random triangular factors and the opening included.
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


def delta(before, after):
    return None if after is None else {k: after[k] - before[k] for k in after}


async def main():
    secint = mpc.SecInt(32, p=P128)
    await mpc.start()
    rng = np.random.default_rng(5)
    a = rng.integers(-2**10, 2**10, size=(6, 6))
    b = rng.integers(-2**10, 2**10, size=(6, 6))
    c = rng.integers(-2**10, 2**10, size=(6, 2))
    s = rng.integers(-2**10, 2**10, size=(3, 4, 4))
    s[1, :, 0] = 0                                  # a singular matrix in the stack
    x = mpc.input(secint.array(a), senders=0)
    y = mpc.input(secint.array(b), senders=0)
    z = mpc.input(secint.array(c), senders=0)
    w = mpc.input(secint.array(s), senders=0)
    await mpc.gather(x, y, z, w)

    before = counters()
    d = mpc.np_det(x)
    await mpc.gather(d)
    det_counts = delta(before, counters())

    # opened products: limb-backed field arrays under install(resident=True)
    A = await mpc.output(x * y, raw=True)
    B = await mpc.output(z * z, raw=True)
    S = await mpc.output(w * w, raw=True)
    before = counters()
    results = [('det', np.linalg.det(A)), ('det stack', np.linalg.det(S)), ('solve', np.linalg.solve(A, B)),
               ('inv', np.linalg.inv(A))]
    results += [(f'matrix_power {e}', np.linalg.matrix_power(A, e)) for e in (-5, 0, 1, 3)]
    public_counts = delta(before, counters())

    print('np_det', int(await mpc.output(d)))
    for name, r in results:
        v = r.value if hasattr(r, 'value') else r
        print(name, np.shape(v), [int(t) for t in np.asarray(v, dtype=object).reshape(-1)])
    if public_counts is not None:
        print('counts public', json.dumps(public_counts))
        print('counts np_det', json.dumps(det_counts))
    await mpc.shutdown()

mpc.run(main())
