"""Times K7 (csrc/reduce.cuh): sums and running sums along an axis, plus np.outer through K1c, on device-resident
operands, against a 2 GiB device copy measured in the same run.

Algorithmic bytes: (O R I + O I) E for a sum, 2 O R I E for a scan (E bytes per element), O I E written for an outer
product.  Prints the card's name and power limit, then one JSON line per shape: best-of CUDA-event time after warm-up,
GB/s and the fraction of the copy rate.  --caller also times one mpc.np_sum(x, axis=1) on a limb-backed (10^4, 10^3)
secint array under install(resident=True), hooked and with its shares settled to Python ints (1 party; needs the
reference, see oracle/reference.py).

    python tools/time_reduce.py [--reps 10] [--caller]
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mpyc_b200                                   # noqa: E402
from mpyc_b200._cabi import lib, check             # noqa: E402
from mpyc_b200.device import DeviceArray, _stream_ptr   # noqa: E402
from stream_probe import card                      # noqa: E402

PRIMES = {1: 2**64 - 189, 2: 2**128 - 173, 4: 2**256 - 189}


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best * 1e-3


def copy_rate(reps):
    n = 2**31 // 8
    a = torch.empty(n, dtype=torch.int64, device='cuda')
    b = torch.empty_like(a)
    return 2 * 2**31 / timed(lambda: b.copy_(a), reps)


def shapes(L):
    """(label, O, R, I) at the byte sizes of 10^8 128-bit elements"""
    n = 2 * 10**8 // L
    return [('full', 1, n, 1), ('cols(n/100,100) axis0', 1, n // 100, 100), ('rows(n/100,100) axis1', n // 100, 100, 1),
            ('(n/3,3) axis0', 1, n // 3, 3), ('(10,n/10) axis1', 10, n // 10, 1)]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--caller', action='store_true')
    a = ap.parse_args()
    print(f'card: {card()}', flush=True)
    copy = copy_rate(a.reps)
    print(json.dumps({'what': 'device copy 2 GiB', 'GBps': round(copy / 1e9, 1)}), flush=True)
    for L, p in PRIMES.items():
        ctx = mpyc_b200.context_for(p)
        E = 8 * L
        n_max = 2 * 10**8 // L
        x = DeviceArray.random(ctx, n_max, seed=1)
        out = DeviceArray.empty(ctx, n_max)
        for label, O, R, I in shapes(L):
            t = timed(lambda: check(lib.mpyc_b200_ff_sum_axis(ctx.handle, x.ptr, O, R, I, None, out.ptr, _stream_ptr())), a.reps)
            nb = (O * R * I + O * I) * E
            print(json.dumps({'op': 'sum', 'L': L, 'shape': label, 'O': O, 'R': R, 'I': I, 'ms': round(t * 1e3, 3),
                              'GBps': round(nb / t / 1e9, 1), 'of_copy': round(nb / t / copy, 3)}), flush=True)
            t = timed(lambda: check(lib.mpyc_b200_ff_cumsum_axis(ctx.handle, x.ptr, O, R, I, 0, out.ptr, _stream_ptr())), a.reps)
            nb = 2 * O * R * I * E
            print(json.dumps({'op': 'cumsum', 'L': L, 'shape': label, 'O': O, 'R': R, 'I': I, 'ms': round(t * 1e3, 3),
                              'GBps': round(nb / t / 1e9, 1), 'of_copy': round(nb / t / copy, 3)}), flush=True)
        del x, out
        torch.cuda.empty_cache()
    ctx = mpyc_b200.context_for(PRIMES[2])
    u, v = DeviceArray.random(ctx, 10**4, seed=2), DeviceArray.random(ctx, 10**4, seed=3)
    c = DeviceArray.empty(ctx, 10**8)
    t = timed(lambda: check(lib.mpyc_b200_ff_matmul(ctx.handle, u.ptr, v.ptr, c.ptr, 10**4, 1, 10**4, _stream_ptr())), a.reps)
    nb = 10**8 * 16
    print(json.dumps({'op': 'outer', 'L': 2, 'shape': '10^4 x 10^4', 'ms': round(t * 1e3, 3), 'GBps': round(nb / t / 1e9, 1),
                      'of_copy': round(nb / t / copy, 3)}), flush=True)
    del c
    if a.caller:
        caller()
    return 0


def caller():
    import numpy as np
    from oracle import reference
    ref = reference.path()
    if ref is None:
        print(json.dumps({'caller': 'skipped: no reference'}))
        return
    sys.path.insert(0, ref)
    sys.argv = [sys.argv[0], '--no-log']
    from mpyc.runtime import mpc
    from mpyc_b200 import install, resident
    install.install(resident=True, operators_min_size=1)
    secint = mpc.SecInt(64)
    mpc.run(mpc.start())
    x = mpc.input(secint.array(np.arange(10**7, dtype=object).reshape(10**4, 10**3) % 1000))[0]
    y = x * x                                          # _reshare: limb-backed shares
    mpc.run(mpc.gather(y))

    def one():
        t0 = time.perf_counter()
        s = mpc.run(mpc.gather(mpc.np_sum(y, axis=1)))
        torch.cuda.synchronize()
        return time.perf_counter() - t0, s
    one()
    hooked, s1 = min((one() for _ in range(3)), key=lambda r: r[0])
    share = y.share.result() if hasattr(y.share, 'result') else y.share
    resident.raw_value(share)._materialise()           # settled: the shares are Python ints, the reference's path
    settled, s2 = one()
    assert [int(v) for v in np.asarray(s1.value).reshape(-1)] == [int(v) for v in np.asarray(s2.value).reshape(-1)]
    print(json.dumps({'caller': 'mpc.np_sum(x, axis=1), (10^4, 10^3) secint, 1 party', 'hooked_ms': round(hooked * 1e3, 2),
                      'settled_ms': round(settled * 1e3, 2)}), flush=True)
    mpc.run(mpc.shutdown())


if __name__ == '__main__':
    sys.exit(main())
