"""Times K10 (csrc/conv.cuh): np.convolve windows of prime-field vectors for L = 1, 2 and 4 (2^61-1, 2^128-173, 2^256-189)
at (2^12, 2^12), (2^16, 2^16) and (2^20, 16) in 'full' mode, (10^4, 10^4 + 1) (np_roll's shape) in 'full' mode and
(2^10, 2^18) in 'valid' mode.  Kernel time is the best-of CUDA-event time of the whole C-ABI call after warm-up (the
split form's scratch and its K7 sum included).  The rate counts the exact products of the window: sum over its outputs of
their number of terms.  In the same run, K1c (k_matmul) at r x k x c = 1024 x 4096 x 1024 (2^32 products) and
64 x 1024 x 256 (2^24), so that the two inner loops are compared at the same product counts.  --caller also times
mpc.np_convolve of two length-4096 secint arrays and mpc.np_roll by a secret shift at N = 4096 under
install(resident=True), 1 party: with the K10 hook and with np.convolve left to the reference on the settled arrays;
both must output the same values.  Prints the card's name and power limit, then one JSON line per measurement.

    python tools/time_conv.py [--reps 5] [--caller]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import mpyc_b200                                   # noqa: E402
from mpyc_b200 import device as dev                # noqa: E402
from mpyc_b200.device import DeviceArray           # noqa: E402
from stream_probe import card                      # noqa: E402

PRIMES = {1: 2**61 - 1, 2: 2**128 - 173, 4: 2**256 - 189}
SHAPES = [(2**12, 2**12, 'full'), (2**16, 2**16, 'full'), (2**20, 16, 'full'), (10**4, 10**4 + 1, 'full'),
          (2**10, 2**18, 'valid')]
MATMULS = [(1024, 4096, 1024), (64, 1024, 256)]


def timed(fn, reps):
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


def window(m, n, mode):
    s, g = min(m, n), max(m, n)
    return {'full': (0, m + n - 1), 'same': ((s - 1) // 2, g), 'valid': (s - 1, g - s + 1)}[mode]


def products(m, n, lo, count):
    k = np.arange(lo, lo + count, dtype=np.int64)
    return int((np.minimum(k, m - 1) - np.maximum(0, k - n + 1) + 1).sum())


def report(**rec):
    print(json.dumps(rec), flush=True)


def kernels(reps):
    for L, p in PRIMES.items():
        ctx = mpyc_b200.context_for(p)
        for m, n, mode in SHAPES:
            a, b = DeviceArray.random(ctx, m, seed=m), DeviceArray.random(ctx, n, seed=n + 1)
            lo, count = window(m, n, mode)
            s = timed(lambda: dev.convolve(ctx, a, m, b, n, lo, count), reps)
            muls = products(m, n, lo, count)
            report(what='convolve', L=L, m=m, n=n, mode=mode, ms=round(s * 1e3, 3), Gmul_per_s=round(muls / s / 1e9, 2))
        for r, k, c in MATMULS:
            A, B = DeviceArray.random(ctx, r * k, seed=r), DeviceArray.random(ctx, k * c, seed=c)
            s = timed(lambda: dev.matmul(ctx, A, B, r, k, c), reps)
            report(what='matmul', L=L, r=r, k=k, c=c, ms=round(s * 1e3, 3), Gmul_per_s=round(r * k * c / s / 1e9, 2))


def caller(N=4096):
    from oracle import reference
    ref = reference.path()
    if ref is None:
        report(what='np_convolve', note='no reference: not measured')
        return
    sys.path.insert(0, ref)
    argv, sys.argv = sys.argv, [sys.argv[0], '--no-log']
    from mpyc.runtime import mpc
    sys.argv = argv
    from mpyc_b200 import install, resident
    install.install(resident=True, operators_min_size=1)
    secint = mpc.SecInt(32)
    mpc.run(mpc.start())
    rng = np.random.default_rng(3)
    x = mpc.input(secint.array(rng.integers(-2**10, 2**10, size=N).astype(object)))[0]
    y = mpc.input(secint.array(rng.integers(-2**10, 2**10, size=N).astype(object)))[0]
    shift = mpc.input(secint(1234))[0]
    mpc.run(mpc.gather(x, y, shift))

    def one(fn):
        t0 = time.perf_counter()
        out = mpc.run(mpc.output(fn()))
        torch.cuda.synchronize()
        return time.perf_counter() - t0, [int(v) for v in out]
    for what, fn in (('np_convolve', lambda: mpc.np_convolve(x, y)), ('np_roll', lambda: mpc.np_roll(x, shift))):
        one(fn)
        hooked, r1 = min((one(fn) for _ in range(3)), key=lambda r: r[0])
        hook, resident.convolve = resident.convolve, lambda *args: resident._MISS   # np.convolve back to the reference
        try:
            settled, r2 = one(fn)
        finally:
            resident.convolve = hook
        assert r1 == r2, what
        report(what=what, N=N, parties=1, hooked_ms=round(hooked * 1e3, 1), settled_ms=round(settled * 1e3, 1))
    mpc.run(mpc.shutdown())


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--caller', action='store_true', help='also the mpc.np_convolve / np_roll measurement')
    a = ap.parse_args()
    print(f'card: {card()}', flush=True)
    kernels(a.reps)
    if a.caller:
        caller()


if __name__ == '__main__':
    main()
